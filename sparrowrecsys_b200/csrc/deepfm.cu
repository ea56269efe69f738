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
#include "deepfm2_layers.cuh"

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
// DeepFM_v2: the tile forward of deepfm2_layers.cuh
// ------------------------------------------------------------------------------------
template <int EP>
__global__ void __launch_bounds__(kThreads) deepfm2_kernel(DeepFm2Params p, BatchView b) {
  using T = DeepFm2Tile<EP, kFmRows>;
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem + T::kXs;
  float* Fs = smem + T::kFs;
  float* H1 = smem + T::kH1;
  float* H2 = smem + T::kH2;
  float* Wds = smem + T::kWds;
  float* Wd1s = smem + T::kWd1s;
  const int row0 = blockIdx.x * kFmRows;
  stage_weights(Wds, p.Wd, 5 * kProj * 32);
  stage_weights(Wd1s, p.Wd1, 32 * 16);
  deepfm2_tile_gather<EP, kFmRows>(p, b, row0, Xs);
  __syncthreads();
  deepfm2_tile_project<EP, kFmRows>(p, Xs, Fs);
  __syncthreads();
  stage_wait();
  __syncthreads();
  deepfm2_tile_mlp<EP, kFmRows>(p, Fs, Wds, Wd1s, H1, H2);
  deepfm2_tile_logits<EP, kFmRows, false>(p, b, row0, Xs, Fs, H2, nullptr, 0, nullptr, [&](int, int row, float z) {
    store_score(b, row, sigmoidf_acc(z));
    if (b.logits) b.logits[row] = z;
  });
}

template <int EP>
static size_t deepfm2_smem() {
  return (size_t)DeepFm2Tile<EP, kFmRows>::kFloats * sizeof(float);
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
