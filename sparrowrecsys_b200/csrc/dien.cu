// dien.cu - DIEN forward (y_pred): gather + GRU + attention + AUGRU + top MLP in one kernel.
//
// Reference: TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DIEN.py:154-256.
//   X = Emb[hist] [T,E], C = Emb[cand] [E]                  (one shared table, :161-167)
//   g_t = GRU(X)_t     Keras GRU, gates z|r|h, reset_after, masked where hist_t == 0 (:169)
//   s_t = sigmoid(Dense1(sigmoid(Dense32(g_t * C))))         attention score (:172-195)
//   u_t = AUGRU(g_t, s_t, u_{t-1})                           three two-layer gates (:204-245)
//   y = sigmoid(Dense1(PReLU(Dense64(PReLU(Dense128([u_T | C | profile | context]))))))
// The AUGRU initial state, a fresh GlorotUniform draw per call in the reference (:235-236),
// is the stored vector `augru_h0` (oracle/ctr_oracle.py::dien_forward states the semantics).
//
// The recurrence is sequential over T and E x E small, so it runs on CUDA cores: one warp
// owns a row, lane e owns element e of every state vector; a matrix-vector product is EP
// shuffle-broadcasts against weight rows held in shared memory (the whole sequence part,
// 15 EP^2 + 45 EP + 68 floats, is staged once per CTA).  GRU step, attention and AUGRU step
// of position t are fused in one loop, so no [T,E] intermediate exists.  The top MLP is the
// 32-row tile code DIN uses (common.cuh::dense_layer).
//
// The AUX variant (dien_kernel<EP, true>) also computes the second output's per-row term, the auxiliary
// head of DIEN.py:261-292 (DESIGN.md section 4.7).  For t = 1..T-1 (1-based positions):
//   pos_t = sigmoid(Dense1_pos(sigmoid(Dense32_pos([g_t | e(h_{t+1})]))))
//   neg_t = sigmoid(Dense1_neg(sigmoid(Dense32_neg([g_t | e(n_{t+1})]))))
//   aux   = sum_t (pos_t + neg_t)             no mask: the slices drop it, padded positions count
// At the kernel's 0-based step t >= 1, h still holds the GRU output of step t-1 while x holds the row of
// hist[t]: they are g_t and e(h_{t+1}) above, and the negative row e(neg[t-1]) is gathered beside x.  Lane
// j owns unit j of both Dense32 layers; their weights (aux_pos_* / aux_neg_*, 2 (64 EP + 66) floats: 16.5 KB
// at EP = 32) are staged after the sequence part.  The plain variant compiles without any of it.
//
// The per-row arithmetic (GRU, attention, AUGRU, auxiliary head) lives in dien_layers.cuh, which the training step
// (dien_train.cu) shares.
#include "dien_layers.cuh"

namespace srs {

template <int EP, bool AUX>
__global__ void __launch_bounds__(kThreads) dien_kernel(DienParams p, BatchView b, DienAuxView ax) {
  static_assert(EP <= 32, "one lane per state element");
  using L = DienBlob<EP>;
  constexpr int R = kDienRows;
  constexpr int KP = 5 * EP + kNumPad;
  constexpr int LDX = KP + 4;
  constexpr int LDH1 = 128 + 4;
  constexpr int LDH2 = 64 + 4;
  // tile column offsets (the order model.cu permutes dense/kernel to)
  constexpr int OFF_UG = 0, OFF_U = EP, OFF_ST = 2 * EP, OFF_C = 3 * EP, OFF_MG = 4 * EP,
                OFF_NUM = 5 * EP;
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;                      // [R][LDX]
  float* H1 = Xs + R * LDX;              // [R][LDH1]
  float* H2 = H1 + R * LDH1;             // [R][LDH2]
  float* Sq = H2 + R * LDH2;             // [L::TOTAL] sequence-part weights
  float* Sa = Sq + L::TOTAL;             // AUX: [DienAuxBlob<EP>::TOTAL] auxiliary-head weights
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int row0 = blockIdx.x * R;

  stage_weights(Sq, p.seq, L::TOTAL);
  if constexpr (AUX) stage_weights(Sa, ax.w, DienAuxBlob<EP>::TOTAL);

  // ---- side features: user genre, user, movie genre rows and numerics ------------
  tile_side_features<EP, R>(Xs, LDX, row0, b, p.user, p.ugenre, p.mgenre, p.n_users, p.n_genres,
                            OFF_UG, OFF_U, OFF_MG, OFF_NUM);
  stage_wait();
  __syncthreads();

  // ---- interest evolution: one warp per row, lane = state element --------------------
  const int le = lane < EP ? lane : EP - 1;          // lanes >= EP mirror lane EP-1 (unused)
  const float att_b = Sq[L::AB + lane], att_wo = Sq[L::AO + lane], att_bo = Sq[L::ABO];
  for (int r = warp; r < R; r += kThreads / 32) {
    const int row = row0 + r;
    float* xrow = Xs + r * LDX;
    if (row >= b.B) {                                      // warp-uniform
      if (lane < EP) { xrow[OFF_C + lane] = 0.f; xrow[OFF_ST + lane] = 0.f; }
      continue;
    }
    // ids pass through float32 numeric columns before the Embedding layer (DIEN.py:96-105)
    int cid = dien_id(__ldg(b.movie_id + row));
    cid = checked_id(cid, p.n_movies, b.err_flag);
    const float c = lane < EP ? __ldg(p.movie + (size_t)cid * EP + lane) : 0.f;
    const int32_t* hrow = b.hist + (size_t)row * b.hist_stride;
    float h = 0.f;                                         // GRU state = its output g_t
    float u = Sq[L::H0 + le];                              // AUGRU state
    int hid_next = __ldg(hrow);
    float aux_row = 0.f;                                   // AUX: sum of pos_t + neg_t
    for (int t = 0; t < p.T; ++t) {
      const int raw = hid_next;
      if (t + 1 < p.T) hid_next = __ldg(hrow + t + 1);
      int hid = dien_id(raw);
      const bool valid = hid != 0;                         // Embedding(mask_zero=True) mask
      hid = checked_id(hid, p.n_movies, b.err_flag);
      const float x = lane < EP ? __ldg(p.movie + (size_t)hid * EP + lane) : 0.f;
      float g_prev = 0.f, xn = 0.f;                        // AUX: g_t and the negative row beside x
      if constexpr (AUX) {
        if (t > 0) {
          g_prev = h;
          int nid = dien_id(__ldg(ax.neg + (size_t)row * ax.neg_stride + t - 1));
          nid = checked_id(nid, p.n_movies, b.err_flag);
          xn = lane < EP ? __ldg(p.movie + (size_t)nid * EP + lane) : 0.f;
        }
      }
      float gz, gr, ghh, grh;
      const float hn = dien_gru_step<EP>(Sq, le, x, h, &gz, &gr, &ghh, &grh);
      if (valid) h = hn;                                   // masked step: state and output carried
      if constexpr (AUX) {
        float sp, sn, pos, neg;
        if (t > 0) aux_row += dien_aux_step<EP>(Sa, g_prev, x, xn, lane, &sp, &sn, &pos, &neg);
      }
      float a;
      const float s = dien_attention<EP>(Sq, lane, h * c, att_b, att_wo, att_bo, &a);
      DienAugruStep st;
      u = dien_augru_step<EP>(Sq, le, h, u, s, &st);
    }
    if (lane < EP) { xrow[OFF_C + lane] = c; xrow[OFF_ST + lane] = u; }
    if constexpr (AUX) {
      if (lane == 0) ax.aux[row] = aux_row;
    }
  }
  __syncthreads();

  // ---- top MLP on the tile ----------------------------------------------------------
  dense_layer<R, 128, 2, 8>(Xs, LDX, KP, p.W1, p.b1, ACT_PRELU, p.a1, H1, LDH1);
  __syncthreads();
  dense_layer<R, 64, 1, 8>(H1, LDH1, 128, p.W2, p.b2, ACT_PRELU, p.a2, H2, LDH2);
  __syncthreads();
  row_dot<R>(H2, LDH2, 64, p.w3, [&](int r, float s) {
    const int row = row0 + r;
    if (row >= b.B) return;
    const float z = s + p.b3;
    store_score(b, row, sigmoidf_acc(z));
    if (b.logits) b.logits[row] = z;
  });
}

// Dynamic shared memory: input tile, two hidden tiles, sequence weights (+ the AUX head's weights).
// EP = 32: 115 088 B plain, 132 000 B AUX.
template <int EP, bool AUX>
static size_t dien_smem() {
  return (size_t)(kDienRows * ((5 * EP + kNumPad + 4) + 132 + 68) + DienBlob<EP>::TOTAL +
                  (AUX ? DienAuxBlob<EP>::TOTAL : 0)) *
         sizeof(float);
}

template <int EP, bool AUX = false>
static cudaError_t launch_dien_t(const DienParams& p, const BatchView& b, cudaStream_t s,
                                 const DienAuxView& a = DienAuxView{}) {
  const int blocks = (b.B + kDienRows - 1) / kDienRows;
  dien_kernel<EP, AUX><<<blocks, kThreads, dien_smem<EP, AUX>(), s>>>(p, b, a);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_dien(const DienParams& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  switch (p.EP) {
    case 12: return launch_dien_t<12>(p, b, s);
    case 16: return launch_dien_t<16>(p, b, s);
    case 32: return launch_dien_t<32>(p, b, s);
  }
  return cudaErrorInvalidValue;
}

cudaError_t launch_dien_aux(const DienParams& p, const DienAuxView& a, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  switch (p.EP) {
    case 12: return launch_dien_t<12, true>(p, b, s, a);
    case 16: return launch_dien_t<16, true>(p, b, s, a);
    case 32: return launch_dien_t<32, true>(p, b, s, a);
  }
  return cudaErrorInvalidValue;
}

// ---- DIEN.py:287: final_loss = binary_crossentropy(y_true, y_pred) - 0.5 * reduce_mean(aux) ----------
constexpr int kFinalThreads = 1024;

// a double summed by every thread of the CTA, reduced in a fixed order (the same bits on every run)
__device__ double cta_sum(double v, double* s_part) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) s_part[warp] = v;
  __syncthreads();
  double t = lane < kFinalThreads / 32 ? s_part[lane] : 0.0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  __syncthreads();                                       // s_part may be reused
  return t;
}

__global__ void __launch_bounds__(kFinalThreads)
dien_final_loss_kernel(const float* __restrict__ logits, const int32_t* __restrict__ labels,
                       const float* __restrict__ aux, int n, float* __restrict__ final_loss, double* sum_dst) {
  __shared__ double s_part[kFinalThreads / 32];
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += kFinalThreads) a += (double)__ldg(aux + i);
  const float half_mean = 0.5f * (float)(cta_sum(a, s_part) / (double)n);   // alpha * reduce_mean, float32
  double f = 0.0;
  for (int i = threadIdx.x; i < n; i += kFinalThreads) {
    const int z = __ldg(labels + i);
    const float v = (z == 0 || z == 1) ? __fsub_rn(logit_bce(__ldg(logits + i), z), half_mean) : NAN;
    final_loss[i] = v;
    f += (double)v;
  }
  if (!sum_dst) return;
  f = cta_sum(f, s_part);
  if (threadIdx.x == 0) *sum_dst = f;
}

cudaError_t launch_dien_final_loss(const float* logits, const int32_t* labels, const float* aux, int n,
                                   float* final_loss, double* sum_dst, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  dien_final_loss_kernel<<<1, kFinalThreads, 0, s>>>(logits, labels, aux, n, final_loss, sum_dst);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t setup_dien_attributes() {
  cudaError_t e;
#define SRS_ATTR(E_, AUX_)                                                                     \
  e = cudaFuncSetAttribute(dien_kernel<E_, AUX_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int)dien_smem<E_, AUX_>());                                        \
  if (e != cudaSuccess) return e;
  SRS_ATTR(12, false) SRS_ATTR(16, false) SRS_ATTR(32, false)
  SRS_ATTR(12, true) SRS_ATTR(16, true) SRS_ATTR(32, true)
#undef SRS_ATTR
  return cudaSuccess;
}

}  // namespace srs
