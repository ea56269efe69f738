// din.cu - DIN forward (CUDA-core variant): gather + activation unit + pooling + top MLP
// in one kernel.
//
// Reference: TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DIN.py:125-167.
//   H = Emb[hist] [T,E], C = Emb[cand] [E]           (one shared table, :132-137)
//   a_t = PReLU_t(Dense32([H_t - C, H_t, C, H_t*C]))  (:141-150, alpha per position)
//   w_t = sigmoid(Dense1(a_t))                        (:151)   sigmoid gate, no softmax
//   pooled = sum_t w_t * H_t                          (:153-158) padding id 0 included
//   y = sigmoid(Dense1(PReLU(Dense64(PReLU(Dense128([profile|pooled|C|context]))))))
//
// The activation-unit Dense is folded algebraically (weights prepared in model.cu):
//   Dense32([h-c, h, c, h*c]) = h.(Wsub+Wh) + (h*c).Wp + c.(Wc-Wsub) + b
//                             = sum_e h[e] * (Wh'[e][j] + c[e] Wp[e][j]) + cst_b[j]
// so per row the 4E-wide concat is never formed and the per-position work drops from
// 4E*32 to E*32 MACs: one warp owns a row, lane j owns activation unit j and keeps the
// folded column M[:, j] in registers; history rows are staged per warp in shared
// memory in chunks and read back as broadcasts.
#include "kernels.h"

namespace srs {

constexpr int kDinRows = 32;     // rows per CTA tile (top MLP tile height)
constexpr int kDinChunk = 32;    // history positions staged per warp at a time

template <int EP>
__global__ void __launch_bounds__(kThreads) din_kernel(DinParams p, BatchView b) {
  constexpr int R = kDinRows;
  constexpr int Q = EP / 4;
  constexpr int KP = 5 * EP + kNumPad;
  constexpr int LDX = KP + 4;
  constexpr int LDH1 = 128 + 4;
  constexpr int LDH2 = 64 + 4;
  constexpr int TC = kDinChunk;
  constexpr int NE = (EP + 31) / 32;            // pooled elements per lane
  // tile column offsets
  constexpr int OFF_UG = 0, OFF_U = EP, OFF_POOL = 2 * EP, OFF_C = 3 * EP, OFF_MG = 4 * EP,
                OFF_NUM = 5 * EP;
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;                      // [R][LDX]
  float* H1 = Xs + R * LDX;              // [R][LDH1]
  float* H2 = H1 + R * LDH1;             // [R][LDH2]
  float* Hc = H2 + R * LDH2;             // [8 warps][TC][EP] history chunk
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int row0 = blockIdx.x * R;
  float* hc = Hc + warp * TC * EP;
  PhaseClock clk(tid == 0);

  // ---- side features: user genre, user, movie genre rows and numerics ------------
  tile_side_features<EP, R>(Xs, LDX, row0, b, p.user, p.ugenre, p.mgenre, p.n_users, p.n_genres,
                            OFF_UG, OFF_U, OFF_MG, OFF_NUM);
  clk.lap(PH_TILE_INPUTS);

  // ---- activation unit + pooling: one warp per row ---------------------------------
  const float wout = __ldg(p.au_wout + lane);
  for (int r = warp; r < R; r += kThreads / 32) {
    const int row = row0 + r;
    float* xrow = Xs + r * LDX;
    if (row >= b.B) {                                      // warp-uniform
      for (int e = lane; e < EP; e += 32) { xrow[OFF_C + e] = 0.f; xrow[OFF_POOL + e] = 0.f; }
      continue;
    }
    // candidate row -> tile (ids pass through float32, DIN.py:95,125)
    int cid = __float2int_rz(__int2float_rn(__ldg(b.movie_id + row)));
    cid = checked_id(cid, p.n_movies, b.err_flag);
    if (lane < Q) *reinterpret_cast<float4*>(xrow + OFF_C + 4 * lane) =
        ldg4(p.movie + (size_t)cid * EP + 4 * lane);
    __syncwarp();
    // folded column of the activation-unit kernel for this row, and its constant
    float M[EP];
    float cst = __ldg(p.au_b + lane);
#pragma unroll
    for (int e = 0; e < EP; ++e) {
      const float c = xrow[OFF_C + e];
      M[e] = fmaf(c, __ldg(p.au_wp + e * 32 + lane), __ldg(p.au_wh + e * 32 + lane));
      cst = fmaf(c, __ldg(p.au_wc + e * 32 + lane), cst);
    }
    clk.lap(PH_W_BUILD);
    float pooled[NE];
#pragma unroll
    for (int n = 0; n < NE; ++n) pooled[n] = 0.f;

    const int32_t* hrow = b.hist + (size_t)row * b.hist_stride;
    for (int t0 = 0; t0 < p.T; t0 += TC) {
      const int nt = min(TC, p.T - t0);
      int hid = 0;
      if (lane < nt) {
        hid = __float2int_rz(__int2float_rn(__ldg(hrow + t0 + lane)));
        hid = checked_id(hid, p.n_movies, b.err_flag);
      }
      __syncwarp();                                         // previous chunk fully consumed
      for (int i0 = 0; i0 < nt * Q; i0 += 32) {             // warp-uniform trip count
        const int i = i0 + lane;
        const int pos = i / Q, q = i % Q;
        const int id = __shfl_sync(0xffffffffu, hid, pos & 31);
        if (i < nt * Q)
          *reinterpret_cast<float4*>(hc + pos * EP + 4 * q) =
              ldg4(p.movie + (size_t)id * EP + 4 * q);
      }
      __syncwarp();
      clk.lap(PH_GATHER_WAIT);
      for (int t = 0; t < nt; ++t) {
        const float* h = hc + t * EP;
        float z0 = cst, z1 = 0.f;
#pragma unroll
        for (int q = 0; q < Q; ++q) {
          const float4 v = *reinterpret_cast<const float4*>(h + 4 * q);
          z0 = fmaf(v.x, M[4 * q], z0);
          z1 = fmaf(v.y, M[4 * q + 1], z1);
          z0 = fmaf(v.z, M[4 * q + 2], z0);
          z1 = fmaf(v.w, M[4 * q + 3], z1);
        }
        float a = z0 + z1;
        a = a > 0.f ? a : __ldg(p.au_alpha + (size_t)(t0 + t) * 32 + lane) * a;
        const float s = warp_sum(a * wout) + p.au_bout;
        const float w = 1.f / (1.f + __expf(-s));
#pragma unroll
        for (int n = 0; n < NE; ++n) {
          const int e = lane + 32 * n;
          if (e < EP) pooled[n] = fmaf(w, h[e], pooled[n]);
        }
      }
      clk.lap(PH_AU_LOOP);
    }
#pragma unroll
    for (int n = 0; n < NE; ++n) {
      const int e = lane + 32 * n;
      if (e < EP) xrow[OFF_POOL + e] = pooled[n];
    }
  }
  clk.lap(PH_AU_LOOP);
  stage_wait();                                            // the side features' copies
  __syncthreads();
  clk.lap(PH_ROW_IMBALANCE);

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
  clk.lap(PH_TOP_MLP);
}

template <int EP>
static size_t din_smem() {
  return (size_t)(kDinRows * ((5 * EP + kNumPad + 4) + 132 + 68) + 8 * kDinChunk * EP) *
         sizeof(float);
}

template <int EP>
static cudaError_t launch_din_t(const DinParams& p, const BatchView& b, cudaStream_t s) {
  const int blocks = (b.B + kDinRows - 1) / kDinRows;
  din_kernel<EP><<<blocks, kThreads, din_smem<EP>(), s>>>(p, b);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_din(const DinParams& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  switch (p.EP) {
    case 12: return launch_din_t<12>(p, b, s);
    case 16: return launch_din_t<16>(p, b, s);
    case 32: return launch_din_t<32>(p, b, s);
    case 64: return launch_din_t<64>(p, b, s);
  }
  return cudaErrorInvalidValue;
}

cudaError_t setup_din_attributes() {
  cudaError_t e;
#define SRS_ATTR(E_)                                                                    \
  e = cudaFuncSetAttribute(din_kernel<E_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int)din_smem<E_>());                                        \
  if (e != cudaSuccess) return e;
  SRS_ATTR(12) SRS_ATTR(16) SRS_ATTR(32) SRS_ATTR(64)
#undef SRS_ATTR
  return cudaSuccess;
}

#ifdef SRS_DIN_PHASES
cudaError_t din_take_phases(unsigned long long* out) { return din_phases_take(out); }
#endif

}  // namespace srs
