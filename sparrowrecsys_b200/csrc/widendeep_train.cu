// widendeep_train.cu - the forward / backward step of Wide&Deep's `model.fit` (WideNDeep.py:99-117) and the
// per-epoch row permutation; the trainer that drives them (dedupe, Adam, metrics) is srs_trainer in trainer.cu.
// DESIGN.md section 4.18.
//
// widendeep_train_step_kernel<EP>: one 32-row tile per CTA, 256 threads.  The forward is embmlp_kernel's
// (embmlp_tile_gather / embmlp_tile_mlp / embmlp_tile_logits of embmlp_layers.cuh), so a step's outputs are the
// serving outputs bit for bit.  The backward runs on the same tile:
//   dz      = (sigmoid(z) - y) / B per row
//   delta2  = dz * w3 where a2 > 0;  delta1 = W2 . delta2 where a1 > 0
//   entries the 10 table rows of each row (a missing genre writes none) with their gradients W1[slot rows] . delta1,
//           and the row's wide row of dense_2/kernel (its crossed bucket, scalar dz), for table_grad_kernel to
//           dedupe in row order
//   partial thread q sums Dense parameter q's gradient over the CTA's rows in row order
// No float atomics.  The trainer's forward for validation and evaluate is embmlp_kernel itself (launch_embmlp).
#include "embmlp_layers.cuh"

namespace srs {

namespace {

constexpr int kWdRows = 32;      // rows per CTA of the step: 4096 rows -> 128 CTAs

// [R][LDX] input | H1, H2, delta1, delta2 [R][LDH] | staged W2 [128][128] | dz [R]
template <int EP>
constexpr int step_smem_floats() {
  return kWdRows * EmbMlpTile<EP>::LDX + 4 * kWdRows * EmbMlpTile<EP>::LDH + 128 * 128 + kWdRows;
}
static_assert(step_smem_floats<64>() * 4 <= 227 * 1024, "the EP = 64 step tile must fit in shared memory");

template <int EP>
__global__ void __launch_bounds__(kThreads) widendeep_train_step_kernel(WideDeepStepArgs a) {
  constexpr int R = kWdRows, LDX = EmbMlpTile<EP>::LDX, LDH = EmbMlpTile<EP>::LDH;
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;
  float* H1 = Xs + R * LDX;
  float* H2 = H1 + R * LDH;
  float* D1 = H2 + R * LDH;                      // delta of the first hidden layer
  float* D2 = D1 + R * LDH;                      // delta of the second
  float* W2s = D2 + R * LDH;
  float* dzs = W2s + 128 * 128;                  // dL/dz
  const EmbMlpBlob ly = EmbMlpBlob::of(EP);
  const BatchView& b = a.io.b;
  const EmbMlpParams& p = a.p;
  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * R;
  const int nv = min(R, b.B - row0);

  stage_weights(W2s, p.W2, 128 * 128);
  embmlp_tile_gather<EP, R>(p, b, row0, Xs);
  stage_wait();
  __syncthreads();
  embmlp_tile_mlp<EP, R, false, true>(p, Xs, p.W1, W2s, H1, H2, LDH);
  embmlp_tile_logits<R>(p, b, row0, H2, LDH, [&](int r, int row, float z, int bucket) {
    const float pr = sigmoidf_acc(z);
    b.probs[row] = pr;
    b.logits[row] = z;
    const float dz = row_dz(pr, __ldg(a.io.label + row), a.io.weight, row, b.B);
    dzs[r] = dz;
    a.io.frow[row] = bucket;
    a.io.fgrad[row] = dz;
  });
  __syncthreads();
  for (int i = tid; i < nv * 128; i += kThreads) {
    const int r = i >> 7, j = i & 127;
    D2[r * LDH + j] = H2[r * LDH + j] > 0.f ? dzs[r] * __ldg(p.w3 + j) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < nv * 128; i += kThreads) {
    const int r = i >> 7, k = i & 127;
    float s = 0.f;
    for (int jj = 0; jj < 128; ++jj) {           // j rotated by k: the lanes of a warp hit distinct banks
      const int j = (jj + k) & 127;
      s = fmaf(W2s[k * 128 + j], D2[r * LDH + j], s);
    }
    D1[r * LDH + k] = H1[r * LDH + k] > 0.f ? s : 0.f;
  }
  __syncthreads();

  // table entries: slot s of tile row r is entry s * B + row
  for (int i = tid; i < nv * kWideDeepTables; i += kThreads) {
    const int r = i / kWideDeepTables, s = i % kWideDeepTables;
    const int row = row0 + r;
    int id;
    if (s < 3) id = __ldg(b.movie_genre + row * 3 + s);
    else if (s == 3) id = __ldg(b.movie_id + row);
    else if (s < 9) id = __ldg(b.user_genre + row * 5 + (s - 4));
    else id = __ldg(b.user_id + row);
    const bool missing = id < 0 || (s != 3 && s != 9 && id >= p.n_genres);
    a.io.trow[s * b.B + row] = missing ? -1 : (int32_t)(a.tab_row0[s] + id);
  }
  // their gradients: tile row q = s * EP + k of W1 against each row's delta1, one warp per q, W1's row read once
  const int warp = tid >> 5, lane = tid & 31;
  for (int q = warp; q < kWideDeepTables * EP; q += kThreads / 32) {
    const float4 w = ldg4(p.W1 + (size_t)q * 128 + 4 * lane);
    const int s = q / EP, k = q % EP;
    for (int r = 0; r < nv; ++r) {
      const float4 d = *reinterpret_cast<const float4*>(D1 + r * LDH + 4 * lane);
      float g = fmaf(w.w, d.w, fmaf(w.z, d.z, fmaf(w.y, d.y, w.x * d.x)));
      g = warp_sum(g);
      if (lane == 0) a.io.gemb[((size_t)s * b.B + row0 + r) * EP + k] = g;
    }
  }

  // Dense gradients of this CTA's rows: parameter q = sum over rows in row order of (input . delta)
  for (int q = tid; q < ly.floats; q += kThreads) {
    const float* in = nullptr;                   // null: the constant 1 (a bias)
    const float* dl = nullptr;                   // null: no gradient (padding)
    int ldi = 0, ldd = 0;
    if (q < ly.b1) { in = Xs + q / 128; ldi = LDX; dl = D1 + q % 128; ldd = LDH; }
    else if (q < ly.W2) { dl = D1 + (q - ly.b1); ldd = LDH; }
    else if (q < ly.b2) { in = H1 + (q - ly.W2) / 128; ldi = LDH; dl = D2 + (q - ly.W2) % 128; ldd = LDH; }
    else if (q < ly.w3) { dl = D2 + (q - ly.b2); ldd = LDH; }
    else if (q < ly.b3) { in = H2 + (q - ly.w3); ldi = LDH; dl = dzs; ldd = 1; }
    else if (q == ly.b3) { dl = dzs; ldd = 1; }
    float s = 0.f;
    if (dl && in) {
      for (int r = 0; r < nv; ++r) s = fmaf(in[r * ldi], dl[r * ldd], s);
    } else if (dl) {
      for (int r = 0; r < nv; ++r) s += dl[r * ldd];
    }
    a.io.part[(size_t)blockIdx.x * ly.floats + q] = s;
  }
}

template <int EP>
cudaError_t launch_step_t(const WideDeepStepArgs* a, cudaStream_t s) {
  constexpr int smem = step_smem_floats<EP>() * (int)sizeof(float);
  if (!a)                                             // the opt-in on the current device, no launch
    return cudaFuncSetAttribute(widendeep_train_step_kernel<EP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  widendeep_train_step_kernel<EP><<<widendeep_train_ctas(a->io.b.B), kThreads, smem, s>>>(*a);
  ++g_launch_count;
  return cudaGetLastError();
}

__global__ void widendeep_permute_kernel(TrainRows src, TrainRows dst, const int32_t* __restrict__ order, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = order[i];
  dst.movie[i] = src.movie[r];
  dst.user[i] = src.user[r];
  dst.rated[i] = src.rated[r];
  dst.label[i] = src.label[r];
  if (src.weight) dst.weight[i] = src.weight[r];
#pragma unroll
  for (int j = 0; j < 3; ++j) dst.mgenre[(size_t)i * 3 + j] = src.mgenre[(size_t)r * 3 + j];
#pragma unroll
  for (int j = 0; j < 5; ++j) dst.ugenre[(size_t)i * 5 + j] = src.ugenre[(size_t)r * 5 + j];
#pragma unroll
  for (int j = 0; j < kNumNumerics; ++j) dst.numerics[(size_t)i * kNumNumerics + j] = src.numerics[(size_t)r * kNumNumerics + j];
}

}  // namespace

int widendeep_train_ctas(int B) { return (B + kWdRows - 1) / kWdRows; }

cudaError_t launch_widendeep_train_step(int EP, const WideDeepStepArgs* a, cudaStream_t s) {
#define SRS_WD_STEP_CASE(E_) \
  if (EP == E_) return launch_step_t<E_>(a, s);
  SRS_WD_STEP_CASE(12) SRS_WD_STEP_CASE(16) SRS_WD_STEP_CASE(32) SRS_WD_STEP_CASE(64)
#undef SRS_WD_STEP_CASE
  return cudaErrorInvalidValue;
}

cudaError_t launch_widendeep_permute(const TrainRows& src, const TrainRows& dst, const int32_t* order, int n,
                                     cudaStream_t s) {
  widendeep_permute_kernel<<<(n + 255) / 256, 256, 0, s>>>(src, dst, order, n);
  ++g_launch_count;
  return cudaGetLastError();
}

}  // namespace srs
