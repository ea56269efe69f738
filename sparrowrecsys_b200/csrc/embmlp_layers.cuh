// embmlp_layers.cuh - the tile forward of EmbeddingMLP and Wide&Deep (EmbeddingMLP.py:72-77, WideNDeep.py:101-107),
// shared by the forward kernel (embmlp.cu, 64-row tiles) and Wide&Deep's training step (widendeep_train.cu, 32-row
// tiles), so that a step's forward is the serving forward bit for bit: every per-row result below depends on the
// row alone, not on the tile's row count.  Tables are padded to EP floats per row; W1 is [KP = 10*EP + 8][128] in
// tile order (movieGenre1..3 | movieId | userGenre1..5 | userId | numerics), W2 [128][128], hidden widths zero
// padded to 128 (EmbMlpBlob, placed by placement.h).
#pragma once

#include "kernels.h"

namespace srs {

template <int EP>
struct EmbMlpTile {
  static constexpr int Q = EP / 4;
  static constexpr int KP = 10 * EP + kNumPad;
  static constexpr int LDX = KP + 4;       // the input tile [R][LDX]
  static constexpr int LDH = 128 + 4;      // a hidden tile [R][LDH]
};

// The input tile of rows row0 .. row0 + R - 1 of b: 10 embedding row gathers (slot-major, 128-bit stores) and the
// 7 numerics (+ one zero).  Rows past the batch end and missing / out-of-vocabulary genres (-1) are zero; an id
// outside its vocabulary latches the error flag.
template <int EP, int R>
__device__ __forceinline__ void embmlp_tile_gather(const EmbMlpParams& p, const BatchView& b, int row0, float* Xs) {
  constexpr int Q = EmbMlpTile<EP>::Q;
  constexpr int LDX = EmbMlpTile<EP>::LDX;
  const int tid = threadIdx.x;
  for (int i = tid; i < R * 10 * Q; i += kThreads) {
    const int q = i % Q;
    const int t = i / Q;
    const int slot = t % 10;
    const int r = t / 10;
    const int row = row0 + r;
    int id = -1;
    const float* table = p.movie;
    if (row < b.B) {
      if (slot < 3) {
        id = __ldg(b.movie_genre + row * 3 + slot);
        table = p.genre[slot];
      } else if (slot == 3) {
        id = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
      } else if (slot < 9) {
        id = __ldg(b.user_genre + row * 5 + (slot - 4));
        table = p.genre[slot - 1];
      } else {
        id = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
        table = p.user;
      }
      if (slot != 3 && slot != 9) {                 // vocabulary column: -1 = missing / OOV
        if (id >= p.n_genres) { atomicExch(b.err_flag, 1); id = -1; }
        if (id < 0) id = -1;
      }
    }
    gather_row<EP>(Xs + r * LDX + slot * EP, table, id, q);
  }
  for (int i = tid; i < R * kNumPad; i += kThreads) {
    const int r = i / kNumPad, j = i % kNumPad;
    const int row = row0 + r;
    float v = 0.f;
    if (j < kNumNumerics && row < b.B) v = __ldg(b.numerics + row * kNumNumerics + j);
    Xs[r * LDX + 10 * EP + j] = v;
  }
}

// The two hidden layers of the tile: H1 = relu(Xs W1 + b1), H2 = relu(H1 W2 + b2) (leading dimension ldh2), on
// CUDA cores; W1 / W2 in shared memory when W1S / W2S, else read in place.  Ends after a barrier.
template <int EP, int R, bool W1S, bool W2S>
__device__ __forceinline__ void embmlp_tile_mlp(const EmbMlpParams& p, const float* Xs, const float* W1,
                                                const float* W2, float* H1, float* H2, int ldh2) {
  constexpr int TM = R / 16;                         // 16 row threads x 16 column threads of 8 columns
  dense_layer<R, 128, TM, 8, W1S>(Xs, EmbMlpTile<EP>::LDX, EmbMlpTile<EP>::KP, W1, p.b1, ACT_RELU, nullptr, H1,
                                  EmbMlpTile<EP>::LDH);
  __syncthreads();
  dense_layer<R, 128, TM, 8, W2S>(H1, EmbMlpTile<EP>::LDH, 128, W2, p.b2, ACT_RELU, nullptr, H2, ldh2);
  __syncthreads();
}

// The logit of each row of the tile that is in the batch: the deep dot, + b3, + (Wide&Deep) the wide weight at
// crossed_bucket(movieId, userRatedMovie1), in that order; emit(r, row, z, bucket) runs on one lane per row
// (bucket -1 for EmbeddingMLP).
template <int R, typename F>
__device__ __forceinline__ void embmlp_tile_logits(const EmbMlpParams& p, const BatchView& b, int row0,
                                                   const float* H2, int ldh, F&& emit) {
  row_dot<R>(H2, ldh, 128, p.w3, [&](int r, float s) {
    const int row = row0 + r;
    if (row >= b.B) return;
    float z = s + __ldg(p.b3);
    int bucket = -1;
    if (p.wide) {
      const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
      const int rated = checked_id(__ldg(b.hist + (size_t)row * b.hist_stride), p.n_movies, b.err_flag);
      bucket = (int)crossed_bucket(mid, rated, (uint32_t)p.cross_buckets);
      z += __ldg(p.wide + bucket);
    }
    emit(r, row, z, bucket);
  });
}

}  // namespace srs
