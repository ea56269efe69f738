// deepfm_layers.cuh - the 32-row tile forward of DeepFM (DeepFM.py:91-113), shared by the forward kernel
// (deepfm.cu) and the training step (deepfm_train.cu), so that a step's forward is the serving forward bit for bit.
// Tables are padded to EP floats per row; W1 is [KP = 2*EP + 8][64] in tile order (deep movie | deep user |
// numerics), W2 [64][64], hidden widths zero-padded to 64 (DeepFmBlob, placed by placement.h).
#pragma once

#include "kernels.h"

namespace srs {

constexpr int kFm1Rows = 32;     // DeepFM tile: 4096 rows -> 128 CTAs

__device__ __forceinline__ int genre_id(const int32_t* col, int row, int stride, int n_genres,
                                        int* err_flag) {
  int id = __ldg(col + row * stride);
  if (id >= n_genres) { atomicExch(err_flag, 1); id = -1; }
  return id < 0 ? -1 : id;
}

// dense_2's four dot weights and its bias, from the blob: in a trainer they change on the device every step, so
// the forward reads them where the step's Adam writes them, with no host read between steps
template <int EP>
__device__ __forceinline__ void deepfm_load_out(DeepFmParams& p) {
  const DeepFmBlob ly = DeepFmBlob::of(EP);
#pragma unroll
  for (int d = 0; d < 4; ++d) p.wdot[d] = __ldg(p.blob + ly.wdot + d);
  p.bout = __ldg(p.blob + ly.bout);
}

// The tile's regions of the kernel's dynamic shared memory (`smem`, which the kernel may extend past kFloats), in
// floats, in this order:
//   Xs  [R][LDX]  deep input: deep_item | deep_user | numerics
//   Fs  [R][LDF]  fm rows: item | user | item_genre | user_genre
//   H1  [R][LDH], H2 [R][LDH]
//   Ds  [R][4]    the four FM dots
//   W1s [KP][64], W2s [64][64]  staged deep kernels
template <int EP>
struct DeepFmTile {
  static constexpr int R = kFm1Rows;
  static constexpr int Q = EP / 4;
  static constexpr int KP = 2 * EP + kNumPad;
  static constexpr int LDX = KP + 4;
  static constexpr int LDF = 4 * EP + 4;
  static constexpr int LDH = 64 + 4;
  static constexpr int kXs = 0;
  static constexpr int kFs = kXs + R * LDX;
  static constexpr int kH1 = kFs + R * LDF;
  static constexpr int kH2 = kH1 + R * LDH;
  static constexpr int kDs = kH2 + R * LDH;
  static constexpr int kW1s = kDs + R * 4;
  static constexpr int kW2s = kW1s + KP * 64;
  static constexpr int kFloats = kW2s + 64 * 64;
};

// Rows row0 .. row0 + 31 of b: gathers, FM dots and the two hidden layers into the tile (ends after a barrier).
template <int EP>
__device__ __forceinline__ void deepfm_tile_forward(const DeepFmParams& p, const BatchView& b, int row0) {
  extern __shared__ __align__(16) float smem[];
  constexpr int R = DeepFmTile<EP>::R;
  constexpr int Q = DeepFmTile<EP>::Q;
  constexpr int KP = DeepFmTile<EP>::KP;
  constexpr int LDX = DeepFmTile<EP>::LDX;
  constexpr int LDF = DeepFmTile<EP>::LDF;
  constexpr int LDH = DeepFmTile<EP>::LDH;
  float* Xs = smem;
  float* Fs = Xs + R * LDX;
  float* H1 = Fs + R * LDF;
  float* H2 = H1 + R * LDH;
  float* Ds = H2 + R * LDH;
  float* W1s = Ds + R * 4;
  float* W2s = W1s + KP * 64;
  const int tid = threadIdx.x;
  stage_weights(W1s, p.W1, KP * 64);
  stage_weights(W2s, p.W2, 64 * 64);

  for (int i = tid; i < R * 6 * Q; i += kThreads) {
    const int q = i % Q;
    const int t = i / Q;
    const int slot = t % 6;
    const int r = t / 6;
    const int row = row0 + r;
    int id = -1;
    const float* table = p.fm_movie;
    float* dst = Fs + r * LDF;
    if (row < b.B) {
      const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
      const int uid = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
      switch (slot) {
        case 0: id = mid; table = p.fm_movie; break;
        case 1: id = uid; table = p.fm_user; break;
        case 2: id = genre_id(b.movie_genre, row, 3, p.n_genres, b.err_flag); table = p.fm_mgenre; break;
        case 3: id = genre_id(b.user_genre, row, 5, p.n_genres, b.err_flag); table = p.fm_ugenre; break;
        case 4: id = mid; table = p.deep_movie; break;
        default: id = uid; table = p.deep_user; break;
      }
    }
    if (slot < 4) dst = Fs + r * LDF + slot * EP;
    else dst = Xs + r * LDX + (slot - 4) * EP;
    gather_row<EP>(dst, table, id, q);
  }
  for (int i = tid; i < R * kNumPad; i += kThreads) {
    const int r = i / kNumPad, j = i % kNumPad;
    const int row = row0 + r;
    float v = 0.f;
    if (j < kNumNumerics && row < b.B) v = __ldg(b.numerics + row * kNumNumerics + j);
    Xs[r * LDX + 2 * EP + j] = v;
  }
  stage_wait();
  __syncthreads();
  if (tid < R * 4) {  // four dots per row (DeepFM.py:100-103): <item,user> <ig,ug> <ig,user> <item,ug>
    const int r = tid >> 2, d = tid & 3;
    const float* f = Fs + r * LDF;
    const float* a = (d == 0 || d == 3) ? f : f + 2 * EP;            // item or item_genre
    const float* c = (d == 0 || d == 2) ? f + EP : f + 3 * EP;       // user or user_genre
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < EP; ++k) s = fmaf(a[k], c[k], s);
    Ds[r * 4 + d] = s;
  }
  dense_layer<R, 64, 1, 8, true>(Xs, LDX, KP, W1s, p.b1, ACT_RELU, nullptr, H1, LDH);
  __syncthreads();
  dense_layer<R, 64, 1, 8, true>(H1, LDH, 64, W2s, p.b2, ACT_RELU, nullptr, H2, LDH);
  __syncthreads();
}

// The logit of each row of the tile that is in the batch: first-order terms, dots, deep dot, bias, in that order;
// emit(r, row, z) runs on one lane per row.
template <int EP, typename F>
__device__ __forceinline__ void deepfm_tile_logits(const DeepFmParams& p, const BatchView& b, int row0,
                                                   F&& emit) {
  extern __shared__ __align__(16) float smem[];
  constexpr int R = DeepFmTile<EP>::R;
  constexpr int LDH = DeepFmTile<EP>::LDH;
  const float* H2 = smem + DeepFmTile<EP>::kH2;
  const float* Ds = smem + DeepFmTile<EP>::kDs;
  row_dot<R>(H2, LDH, 64, p.wdeep, [&](int r, float s) {
    const int row = row0 + r;
    if (row >= b.B) return;
    const int G = p.n_genres;
    const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
    const int uid = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
    const int ig = genre_id(b.movie_genre, row, 3, G, b.err_flag);
    const int ug = genre_id(b.user_genre, row, 5, G, b.err_flag);
    // one-hot block order (sorted column names): movieGenre1 | movieId | userGenre1 | userId
    float z = 0.f;
    if (ig >= 0) z += __ldg(p.first + ig);
    z += __ldg(p.first + G + mid);
    if (ug >= 0) z += __ldg(p.first + G + p.n_movies + ug);
    z += __ldg(p.first + (size_t)(2 * G + p.n_movies) + uid);
#pragma unroll
    for (int d = 0; d < 4; ++d) z = fmaf(Ds[r * 4 + d], p.wdot[d], z);
    z += s + p.bout;
    emit(r, row, z);
  });
}

}  // namespace srs
