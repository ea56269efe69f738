// deepfm.cu - DeepFM (pairwise-dot FM) and DeepFM_v2 (sum-square FM) forward.
//
// Reference: DeepFM.py:91-113 and DeepFM_v2.py:98-155
// (TFRecModel/src/com/sparrowrecsys/offline/tensorflow/).
//
// The reference materialises a [B, 31040] one-hot block and multiplies it by a
// Dense(1) kernel; that product is four scalar gathers W[offset + id], which is how
// both kernels evaluate the first-order term.  Everything else per 64-row tile:
// row gathers straight into shared memory, FM interaction on the tile, the deep MLP
// with register-tiled FFMA, one score per row out.
#include "deepfm_layers.cuh"

namespace srs {

constexpr int kFmRows = 64;      // DeepFM_v2 tile

// ------------------------------------------------------------------------------------
// DeepFM (v1): the tile forward of deepfm_layers.cuh
// ------------------------------------------------------------------------------------
template <int EP>
__global__ void __launch_bounds__(kThreads) deepfm_kernel(DeepFmParams p, BatchView b) {
  const int row0 = blockIdx.x * kFm1Rows;
  deepfm_tile_forward<EP>(p, b, row0);
  deepfm_load_out<EP>(p);                 // after the forward: the five floats are not held across its tiles
  deepfm_tile_logits<EP>(p, b, row0, [&](int, int row, float z) {
    store_score(b, row, sigmoidf_acc(z));
    if (b.logits) b.logits[row] = z;
  });
}

template <int EP>
static size_t deepfm_smem() {
  return (size_t)DeepFmTile<EP>::kFloats * sizeof(float);
}

template <int EP>
static cudaError_t launch_deepfm_t(const DeepFmParams& p, const BatchView& b, cudaStream_t s) {
  const int blocks = (b.B + kFm1Rows - 1) / kFm1Rows;
  deepfm_kernel<EP><<<blocks, kThreads, deepfm_smem<EP>(), s>>>(p, b);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_deepfm(const DeepFmParams& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  switch (p.EP) {
    case 12: return launch_deepfm_t<12>(p, b, s);
    case 16: return launch_deepfm_t<16>(p, b, s);
    case 32: return launch_deepfm_t<32>(p, b, s);
    case 64: return launch_deepfm_t<64>(p, b, s);
  }
  return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------
// DeepFM_v2
// ------------------------------------------------------------------------------------
constexpr int kProj = 64;      // per-field projection width (DeepFM_v2.py:114)

template <int EP>
__global__ void __launch_bounds__(kThreads) deepfm2_kernel(DeepFm2Params p, BatchView b) {
  constexpr int R = kFmRows;
  constexpr int Q = EP / 4;
  constexpr int KX = 4 * EP + kNumPad;
  constexpr int LDX = KX + 4;
  constexpr int LDF = 5 * kProj + 4;
  constexpr int LD1 = 32 + 4;
  constexpr int LD2 = 16 + 4;
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;                 // [R][LDX]  item_genre | movie | user_genre | user | numerics
  float* Fs = Xs + R * LDX;         // [R][LDF]  five projected fields (DeepFM_v2.py:121)
  float* D1 = Fs + R * LDF;         // [R][LD1]
  float* D2 = D1 + R * LD1;         // [R][LD2]
  float* Wds = D2 + R * LD2;        // [320][32] staged deep kernel
  float* Wd1s = Wds + 5 * kProj * 32;   // [32][16]
  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * R;
  stage_weights(Wds, p.Wd, 5 * kProj * 32);
  stage_weights(Wd1s, p.Wd1, 32 * 16);

  for (int i = tid; i < R * 4 * Q; i += kThreads) {
    const int q = i % Q;
    const int t = i / Q;
    const int slot = t % 4;
    const int r = t / 4;
    const int row = row0 + r;
    int id = -1;
    const float* table = p.movie;
    if (row < b.B) {
      switch (slot) {
        case 0: id = genre_id(b.movie_genre, row, 3, p.n_genres, b.err_flag); table = p.mgenre; break;
        case 1: id = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag); table = p.movie; break;
        case 2: id = genre_id(b.user_genre, row, 5, p.n_genres, b.err_flag); table = p.ugenre; break;
        default: id = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag); table = p.user; break;
      }
    }
    gather_row<EP>(Xs + r * LDX + slot * EP, table, id, q);
  }
  for (int i = tid; i < R * kNumPad; i += kThreads) {
    const int r = i / kNumPad, j = i % kNumPad;
    const int row = row0 + r;
    float v = 0.f;
    if (j < kNumNumerics && row < b.B) v = __ldg(b.numerics + row * kNumNumerics + j);
    Xs[r * LDX + 4 * EP + j] = v;
  }
  __syncthreads();
#pragma unroll
  for (int f = 0; f < 4; ++f)
    dense_layer<R, kProj, 2, 8>(Xs + f * EP, LDX, EP, p.proj[f], p.proj_b[f], ACT_NONE, nullptr,
                                Fs + f * kProj, LDF);
  dense_layer<R, kProj, 2, 8>(Xs + 4 * EP, LDX, kNumPad, p.proj_num, p.proj_num_b, ACT_NONE,
                              nullptr, Fs + 4 * kProj, LDF);
  __syncthreads();
  stage_wait();
  __syncthreads();
  dense_layer<R, 32, 1, 8, true>(Fs, LDF, 5 * kProj, Wds, p.bd, ACT_RELU, nullptr, D1, LD1);
  __syncthreads();
  dense_layer<R, 16, 1, 4, true>(D1, LD1, 32, Wd1s, p.bd1, ACT_RELU, nullptr, D2, LD2);
  __syncthreads();

  const int warp = tid >> 5, lane = tid & 31;
  for (int r = warp; r < R; r += kThreads / 32) {
    const int row = row0 + r;
    if (row >= b.B) continue;                      // warp-uniform
    float part = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {                  // FM: (sum_f v)^2 - sum_f v^2, no 1/2 (:147-152)
      const int c = lane + 32 * h;
      float s = 0.f, q2 = 0.f;
#pragma unroll
      for (int f = 0; f < 5; ++f) {
        const float v = Fs[r * LDF + f * kProj + c];
        s += v;
        q2 = fmaf(v, v, q2);
      }
      part = fmaf(s * s - q2, __ldg(p.wout + 1 + c), part);
    }
    if (lane < 16) part = fmaf(D2[r * LD2 + lane], __ldg(p.wout + 1 + kProj + lane), part);
    if (lane == 0) {                               // first-order term (:98-104)
      const int G = p.n_genres;
      const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
      const int uid = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
      const int ig = genre_id(b.movie_genre, row, 3, G, b.err_flag);
      const int ug = genre_id(b.user_genre, row, 5, G, b.err_flag);
      float first = p.first_bias;
      if (ig >= 0) first += __ldg(p.first + ig);
      first += __ldg(p.first + G + mid);
      if (ug >= 0) first += __ldg(p.first + G + p.n_movies + ug);
      first += __ldg(p.first + (size_t)(2 * G + p.n_movies) + uid);
#pragma unroll
      for (int j = 0; j < kNumNumerics; ++j)
        first = fmaf(Xs[r * LDX + 4 * EP + j], __ldg(p.first_num + j), first);
      part = fmaf(first, __ldg(p.wout), part);
    }
    const float z = warp_sum(part) + p.bout;
    if (lane == 0) {
      store_score(b, row, sigmoidf_acc(z));
      if (b.logits) b.logits[row] = z;
    }
  }
}

template <int EP>
static size_t deepfm2_smem() {
  return ((size_t)kFmRows * ((4 * EP + kNumPad + 4) + (5 * kProj + 4) + 36 + 20) + 5 * kProj * 32 + 32 * 16) *
         sizeof(float);
}

template <int EP>
static cudaError_t launch_deepfm2_t(const DeepFm2Params& p, const BatchView& b, cudaStream_t s) {
  const int blocks = (b.B + kFmRows - 1) / kFmRows;
  deepfm2_kernel<EP><<<blocks, kThreads, deepfm2_smem<EP>(), s>>>(p, b);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_deepfm2(const DeepFm2Params& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  switch (p.EP) {
    case 12: return launch_deepfm2_t<12>(p, b, s);
    case 16: return launch_deepfm2_t<16>(p, b, s);
    case 32: return launch_deepfm2_t<32>(p, b, s);
    case 64: return launch_deepfm2_t<64>(p, b, s);
  }
  return cudaErrorInvalidValue;
}

cudaError_t setup_deepfm_attributes() {
  cudaError_t e;
#define SRS_ATTR(E_)                                                                       \
  e = cudaFuncSetAttribute(deepfm_kernel<E_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int)deepfm_smem<E_>());                                        \
  if (e != cudaSuccess) return e;                                                          \
  e = cudaFuncSetAttribute(deepfm2_kernel<E_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int)deepfm2_smem<E_>());                                       \
  if (e != cudaSuccess) return e;
  SRS_ATTR(12) SRS_ATTR(16) SRS_ATTR(32) SRS_ATTR(64)
#undef SRS_ATTR
  return cudaSuccess;
}

}  // namespace srs
