// deepfm_train.cu - the forward / backward step of DeepFM's `model.fit` (DeepFM.py) and the per-epoch row
// permutation; the trainer that drives them (dedupe, Adam, metrics) is srs_trainer in trainer.cu.
// DESIGN.md section 4.9.
//
// deepfm_train_step_kernel<EP>: one 32-row tile per CTA, 256 threads.  The forward is deepfm_kernel's
// (deepfm_tile_forward / deepfm_tile_logits of deepfm_layers.cuh), so a step's outputs are the serving outputs
// bit for bit.  The backward runs on the same tile:
//   dz      = (sigmoid(z) - y) / B per row
//   delta2  = dz * wdeep where a2 > 0;  delta1 = W2 . delta2 where a1 > 0
//   entries the 6 table rows of each row (4 FM, 2 deep; a missing genre writes none) with their gradients, and
//           the 4 one-hot rows of dense_2/kernel (scalar dz), for table_grad_kernel to dedupe in row order
//   partial thread q sums Dense parameter q's gradient over the CTA's rows in row order
// No float atomics.  The trainer's forward for validation and evaluate is deepfm_kernel itself (launch_deepfm).
#include "deepfm_layers.cuh"

namespace srs {

namespace {

template <int EP>
constexpr int step_smem_floats() {
  return DeepFmTile<EP>::kFloats + 2 * kFm1Rows * DeepFmTile<EP>::LDH + kFm1Rows;   // + delta1, delta2, dz
}

template <int EP>
__global__ void __launch_bounds__(kThreads) deepfm_train_step_kernel(DeepFmStepArgs a) {
  using T = DeepFmTile<EP>;
  constexpr int R = T::R, LDX = T::LDX, LDF = T::LDF, LDH = T::LDH;
  extern __shared__ __align__(16) float smem[];
  const float* Xs = smem + T::kXs;
  const float* Fs = smem + T::kFs;
  const float* H1 = smem + T::kH1;
  const float* H2 = smem + T::kH2;
  const float* Ds = smem + T::kDs;
  const float* W1s = smem + T::kW1s;
  const float* W2s = smem + T::kW2s;
  float* D1 = smem + T::kFloats;                 // [R][LDH] delta of the first hidden layer
  float* D2 = D1 + R * LDH;                      // [R][LDH] delta of the second
  float* dzs = D2 + R * LDH;                     // [R]      dL/dz
  const DeepFmBlob ly = DeepFmBlob::of(EP);
  const BatchView& b = a.io.b;
  DeepFmParams p = a.p;
  deepfm_load_out<EP>(p);
  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * R;
  const int nv = min(R, b.B - row0);

  deepfm_tile_forward<EP>(p, b, row0);
  deepfm_tile_logits<EP>(p, b, row0, [&](int r, int row, float z) {
    const float pr = sigmoidf_acc(z);
    b.probs[row] = pr;
    b.logits[row] = z;
    dzs[r] = row_dz(pr, __ldg(a.io.label + row), a.io.weight, row, b.B);
  });
  __syncthreads();
  for (int i = tid; i < nv * 64; i += kThreads) {
    const int r = i >> 6, j = i & 63;
    D2[r * LDH + j] = H2[r * LDH + j] > 0.f ? dzs[r] * __ldg(p.wdeep + j) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < nv * 64; i += kThreads) {
    const int r = i >> 6, k = i & 63;
    float s = 0.f;
    for (int jj = 0; jj < 64; ++jj) {           // j rotated by k: the lanes of a warp hit distinct banks
      const int j = (jj + k) & 63;
      s = fmaf(W2s[k * 64 + j], D2[r * LDH + j], s);
    }
    D1[r * LDH + k] = H1[r * LDH + k] > 0.f ? s : 0.f;
  }
  __syncthreads();

  // table entries: slot s of tile row r is entry s * B + row
  for (int i = tid; i < nv * kDeepFmTables; i += kThreads) {
    const int r = i / kDeepFmTables, s = i % kDeepFmTables;
    const int row = row0 + r;
    int id;
    switch (s) {
      case 0: case 4: id = __ldg(b.movie_id + row); break;
      case 1: case 5: id = __ldg(b.user_id + row); break;
      case 2: id = __ldg(b.movie_genre + row * 3); break;
      default: id = __ldg(b.user_genre + row * 5); break;
    }
    a.io.trow[s * b.B + row] = id < 0 ? -1 : (int32_t)(a.tab_row0[s] + id);
    if (s < 4) {                                 // the one-hot rows: movieGenre1 | movieId | userGenre1 | userId
      const int G = p.n_genres;                  // slot s: movieId, userId, movieGenre1, userGenre1
      const int off = s == 0 ? G : s == 1 ? 2 * G + p.n_movies : s == 2 ? 0 : G + p.n_movies;
      a.io.frow[s * b.B + row] = id < 0 ? -1 : off + id;
      a.io.fgrad[s * b.B + row] = dzs[r];
    }
  }
  const float w0 = p.wdot[0], w1 = p.wdot[1], w2 = p.wdot[2], w3 = p.wdot[3];
  for (int i = tid; i < nv * kDeepFmTables * EP; i += kThreads) {
    const int k = i % EP, t = i / EP;
    const int s = t % kDeepFmTables, r = t / kDeepFmTables;
    const float* f = Fs + r * LDF;               // item | user | item_genre | user_genre
    const float dz = dzs[r];
    float g;
    if (s < 4) {                                 // each FM row: dz * sum(dot weight * the other factor)
      const float item = f[k], user = f[EP + k], ig = f[2 * EP + k], ug = f[3 * EP + k];
      switch (s) {
        case 0: g = dz * (w0 * user + w3 * ug); break;
        case 1: g = dz * (w0 * item + w2 * ig); break;
        case 2: g = dz * (w1 * ug + w2 * user); break;
        default: g = dz * (w1 * ig + w3 * item); break;
      }
    } else {                                     // the deep rows: W1 . delta1 at the row's tile columns
      const float* w = W1s + ((s - 4) * EP + k) * 64;
      const float* d1 = D1 + r * LDH;
      g = 0.f;
      for (int jj = 0; jj < 64; ++jj) {
        const int j = (jj + k) & 63;
        g = fmaf(w[j], d1[j], g);
      }
    }
    a.io.gemb[((size_t)s * b.B + row0 + r) * EP + k] = g;
  }

  // Dense gradients of this CTA's rows: parameter q = sum over rows in row order of (input . delta)
  for (int q = tid; q < ly.floats; q += kThreads) {
    const float* in = nullptr;                   // null: the constant 1 (a bias)
    const float* dl = nullptr;                   // null: no gradient (padding)
    int ldi = 0, ldd = 0;
    if (q < ly.b1) { in = Xs + q / 64; ldi = LDX; dl = D1 + q % 64; ldd = LDH; }
    else if (q < ly.W2) { dl = D1 + (q - ly.b1); ldd = LDH; }
    else if (q < ly.b2) { in = H1 + (q - ly.W2) / 64; ldi = LDH; dl = D2 + (q - ly.W2) % 64; ldd = LDH; }
    else if (q < ly.wdeep) { dl = D2 + (q - ly.b2); ldd = LDH; }
    else if (q < ly.wdot) { in = H2 + (q - ly.wdeep); ldi = LDH; dl = dzs; ldd = 1; }
    else if (q < ly.bout) { in = Ds + (q - ly.wdot); ldi = 4; dl = dzs; ldd = 1; }
    else if (q == ly.bout) { dl = dzs; ldd = 1; }
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
cudaError_t launch_step_t(const DeepFmStepArgs* a, cudaStream_t s) {
  constexpr int smem = step_smem_floats<EP>() * (int)sizeof(float);
  if (!a)                                             // the opt-in on the current device, no launch
    return cudaFuncSetAttribute(deepfm_train_step_kernel<EP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  deepfm_train_step_kernel<EP><<<deepfm_train_ctas(a->io.b.B), kThreads, smem, s>>>(*a);
  ++g_launch_count;
  return cudaGetLastError();
}

__global__ void deepfm_permute_kernel(TrainRows src, TrainRows dst, const int32_t* __restrict__ order, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = order[i];
  dst.movie[i] = src.movie[r];
  dst.user[i] = src.user[r];
  dst.mgenre[(size_t)i * 3] = src.mgenre[(size_t)r * 3];
  dst.ugenre[(size_t)i * 5] = src.ugenre[(size_t)r * 5];
  dst.label[i] = src.label[r];
  if (src.weight) dst.weight[i] = src.weight[r];
#pragma unroll
  for (int j = 0; j < kNumNumerics; ++j) dst.numerics[(size_t)i * kNumNumerics + j] = src.numerics[(size_t)r * kNumNumerics + j];
}

}  // namespace

int deepfm_train_ctas(int B) { return (B + kFm1Rows - 1) / kFm1Rows; }

cudaError_t launch_deepfm_train_step(int EP, const DeepFmStepArgs* a, cudaStream_t s) {
#define SRS_DEEPFM_TRAIN_CASE(E_) \
  if (EP == E_) return launch_step_t<E_>(a, s);
  SRS_DEEPFM_TRAIN_CASE(12) SRS_DEEPFM_TRAIN_CASE(16) SRS_DEEPFM_TRAIN_CASE(32) SRS_DEEPFM_TRAIN_CASE(64)
#undef SRS_DEEPFM_TRAIN_CASE
  return cudaErrorInvalidValue;
}

cudaError_t launch_deepfm_permute(const TrainRows& src, const TrainRows& dst, const int32_t* order, int n,
                                  cudaStream_t s) {
  deepfm_permute_kernel<<<(n + 255) / 256, 256, 0, s>>>(src, dst, order, n);
  ++g_launch_count;
  return cudaGetLastError();
}

}  // namespace srs
