// embmlp.cu - EmbeddingMLP and Wide&Deep forward, one fused kernel.
//
// Reference: EmbeddingMLP.py:72-77 and WideNDeep.py:101-107
// (TFRecModel/src/com/sparrowrecsys/offline/tensorflow/).  Per row: 10 embedding row
// gathers (8 genre slots + movieId + userId) and 7 numerics form the Dense input;
// Dense(128,relu) -> Dense(128,relu) -> Dense(1,sigmoid).  Wide&Deep adds one scalar
// weight gathered at hash(movieId x userRatedMovie1) % 10000 before the sigmoid
// (the one-hot x Dense(1) product of the reference collapses to that gather).
//
// A CTA owns a tile of 64 rows: the gathers land directly in the shared-memory
// input tile (slot-major, 128-bit stores), the three Dense layers run on the tile
// with register-tiled FFMA, only the scores leave the SM.  The tile forward is
// embmlp_layers.cuh's, shared with Wide&Deep's training step.
#include "embmlp_layers.cuh"

namespace srs {

constexpr int kEmbRows = 64;

template <int EP>
__global__ void __launch_bounds__(kThreads) embmlp_kernel(EmbMlpParams p, BatchView b) {
  constexpr int R = kEmbRows;
  constexpr int KP = EmbMlpTile<EP>::KP;
  constexpr int LDX = EmbMlpTile<EP>::LDX;
  constexpr int LDH = EmbMlpTile<EP>::LDH;
  static_assert(LDX >= LDH, "second hidden tile aliases the input tile");
  constexpr bool STAGE_W1 = EP == 12;      // 64 KB: fits next to the tiles only for the reference shape
  constexpr bool STAGE_W2 = EP <= 32;      // 64 KB
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;
  float* H1 = smem + R * LDX;
  float* W2s = H1 + R * LDH;               // [128][128] if STAGE_W2
  float* W1s = W2s + (STAGE_W2 ? 128 * 128 : 0);   // [KP][128] if STAGE_W1
  const int row0 = blockIdx.x * R;
  if (STAGE_W1) stage_weights(W1s, p.W1, KP * 128);
  if (STAGE_W2) stage_weights(W2s, p.W2, 128 * 128);

  embmlp_tile_gather<EP, R>(p, b, row0, Xs);
  if (STAGE_W1 || STAGE_W2) stage_wait();
  __syncthreads();
  float* H2 = Xs;
  embmlp_tile_mlp<EP, R, STAGE_W1, STAGE_W2>(p, Xs, STAGE_W1 ? W1s : p.W1, STAGE_W2 ? W2s : p.W2, H1, H2, LDX);
  embmlp_tile_logits<R>(p, b, row0, H2, LDX, [&](int, int row, float z, int) {
    store_score(b, row, sigmoidf_acc(z));
    if (b.logits) b.logits[row] = z;
  });
}

template <int EP>
static size_t embmlp_smem() {
  size_t floats = (size_t)kEmbRows * ((10 * EP + kNumPad + 4) + 132);
  if (EP <= 32) floats += 128 * 128;                         // staged W2
  if (EP == 12) floats += (size_t)(10 * EP + kNumPad) * 128;  // staged W1
  return floats * sizeof(float);
}

template <int EP>
static cudaError_t launch_embmlp_t(const EmbMlpParams& p, const BatchView& b, cudaStream_t s) {
  const int blocks = (b.B + kEmbRows - 1) / kEmbRows;
  embmlp_kernel<EP><<<blocks, kThreads, embmlp_smem<EP>(), s>>>(p, b);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_embmlp(const EmbMlpParams& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  switch (p.EP) {
    case 12: return launch_embmlp_t<12>(p, b, s);
    case 16: return launch_embmlp_t<16>(p, b, s);
    case 32: return launch_embmlp_t<32>(p, b, s);
    case 64: return launch_embmlp_t<64>(p, b, s);
  }
  return cudaErrorInvalidValue;
}

cudaError_t setup_embmlp_attributes() {
  cudaError_t e;
#define SRS_ATTR(E_)                                                                   \
  e = cudaFuncSetAttribute(embmlp_kernel<E_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int)embmlp_smem<E_>());                                    \
  if (e != cudaSuccess) return e;
  SRS_ATTR(12) SRS_ATTR(16) SRS_ATTR(32) SRS_ATTR(64)
#undef SRS_ATTR
  return cudaSuccess;
}

}  // namespace srs
