// deepfm2_layers.cuh - the tile forward of DeepFM_v2 (DeepFM_v2.py:98-155), shared by the forward kernel
// (deepfm.cu, 64-row tiles) and DeepFM_v2's training step (deepfm2_train.cu, 32-row tiles), so that a step's
// forward is the serving forward bit for bit: every per-row result below depends on the row alone, not on the
// tile's row count.  Tables are padded to EP floats per row; the Dense weights are one DeepFm2Blob (placement.h).
#pragma once

#include "deepfm_layers.cuh"

namespace srs {

constexpr int kProj = 64;      // per-field projection width (DeepFM_v2.py:114)

// The tile's regions of the kernel's dynamic shared memory (`smem`, which the step extends past kFloats), in
// floats, in this order:
//   Xs  [R][LDX]  item_genre | movie | user_genre | user | numerics
//   Fs  [R][LDF]  the five projected fields (DeepFM_v2.py:121)
//   H1  [R][LD1], H2 [R][LD2]  the deep MLP's hidden layers
//   Wds [320][32], Wd1s [32][16]  staged deep kernels
template <int EP, int R_>
struct DeepFm2Tile {
  static constexpr int R = R_;
  static constexpr int Q = EP / 4;
  static constexpr int KX = 4 * EP + kNumPad;
  static constexpr int LDX = KX + 4;
  static constexpr int LDF = 5 * kProj + 4;
  static constexpr int LD1 = 32 + 4;
  static constexpr int LD2 = 16 + 4;
  static constexpr int kXs = 0;
  static constexpr int kFs = kXs + R * LDX;
  static constexpr int kH1 = kFs + R * LDF;
  static constexpr int kH2 = kH1 + R * LD1;
  static constexpr int kWds = kH2 + R * LD2;
  static constexpr int kWd1s = kWds + 5 * kProj * 32;
  static constexpr int kFloats = kWd1s + 32 * 16;
};

// The input tile of rows row0 .. row0 + R - 1 of b: the four embedding rows (128-bit stores) and the 7 numerics
// (+ one zero).  Rows past the batch end and missing genres are zero; an id outside its vocabulary latches the
// error flag.
template <int EP, int R>
__device__ __forceinline__ void deepfm2_tile_gather(const DeepFm2Params& p, const BatchView& b, int row0, float* Xs) {
  constexpr int Q = DeepFm2Tile<EP, R>::Q;
  constexpr int LDX = DeepFm2Tile<EP, R>::LDX;
  const int tid = threadIdx.x;
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
}

// The five projected fields of the tile: Fs[r][f * 64 + c] = x_f . proj_f[:, c] + proj_f/bias[c]
template <int EP, int R>
__device__ __forceinline__ void deepfm2_tile_project(const DeepFm2Params& p, const float* Xs, float* Fs) {
  constexpr int LDX = DeepFm2Tile<EP, R>::LDX;
  constexpr int LDF = DeepFm2Tile<EP, R>::LDF;
#pragma unroll
  for (int f = 0; f < 4; ++f)
    dense_layer<R, kProj, R / 32, 8>(Xs + f * EP, LDX, EP, p.proj[f], p.proj_b[f], ACT_NONE, nullptr,
                                     Fs + f * kProj, LDF);
  dense_layer<R, kProj, R / 32, 8>(Xs + 4 * EP, LDX, kNumPad, p.proj_num, p.proj_num_b, ACT_NONE, nullptr,
                                   Fs + 4 * kProj, LDF);
}

// The deep MLP over Flatten(Fs) with the staged kernels: H1 = relu(Fs Wd + bd), H2 = relu(H1 Wd1 + bd1).  Each
// output is fmaf over k in order from 0, then + bias, then relu, whatever the tiling: a 32-row tile, which
// dense_layer cannot spread over 256 threads at width 16, computes H2 element by element in that order.  Ends
// after a barrier.
template <int EP, int R>
__device__ __forceinline__ void deepfm2_tile_mlp(const DeepFm2Params& p, const float* Fs, const float* Wds,
                                                 const float* Wd1s, float* H1, float* H2) {
  constexpr int LDF = DeepFm2Tile<EP, R>::LDF;
  constexpr int LD1 = DeepFm2Tile<EP, R>::LD1;
  constexpr int LD2 = DeepFm2Tile<EP, R>::LD2;
  dense_layer<R, 32, 1, R / 8, true>(Fs, LDF, 5 * kProj, Wds, p.bd, ACT_RELU, nullptr, H1, LD1);
  __syncthreads();
  if constexpr (R == 64) {
    dense_layer<R, 16, 1, 4, true>(H1, LD1, 32, Wd1s, p.bd1, ACT_RELU, nullptr, H2, LD2);
  } else {
    for (int i = threadIdx.x; i < R * 16; i += kThreads) {
      const int r = i >> 4, j = i & 15;
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 32; ++k) acc = fmaf(H1[r * LD1 + k], Wd1s[k * 16 + j], acc);
      H2[r * LD2 + j] = fmaxf(acc + __ldg(p.bd1 + j), 0.f);
    }
  }
  __syncthreads();
}

// The logit of each row of the tile that is in the batch, one warp per row: the FM terms (sum_f F)^2 - sum_f F^2
// (no 1/2, DeepFM_v2.py:147-152) and the deep rows against out/kernel, then the first-order term (:98-104) on lane
// 0, the warp's sum and out/bias.  The first-order bias is first_cat/bias + first_num/bias, one float add.
// emit(r, row, z) runs on lane 0.  KEEP (the training step): also FMs[r][c] = the FM term c and firsts[r] = the
// first-order value, which out/kernel's gradient needs.
template <int EP, int R, bool KEEP, typename F>
__device__ __forceinline__ void deepfm2_tile_logits(const DeepFm2Params& p, const BatchView& b, int row0,
                                                    const float* Xs, const float* Fs, const float* H2, float* FMs,
                                                    int ldm, float* firsts, F&& emit) {
  constexpr int LDX = DeepFm2Tile<EP, R>::LDX;
  constexpr int LDF = DeepFm2Tile<EP, R>::LDF;
  constexpr int LD2 = DeepFm2Tile<EP, R>::LD2;
  const DeepFm2Blob ly = DeepFm2Blob::of(EP);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < R; r += kThreads / 32) {
    const int row = row0 + r;
    if (row >= b.B) continue;                      // warp-uniform
    float part = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = lane + 32 * h;
      float s = 0.f, q2 = 0.f;
#pragma unroll
      for (int f = 0; f < 5; ++f) {
        const float v = Fs[r * LDF + f * kProj + c];
        s += v;
        q2 = fmaf(v, v, q2);
      }
      const float fm = s * s - q2;
      if (KEEP) FMs[r * ldm + c] = fm;
      part = fmaf(fm, __ldg(p.wout + 1 + c), part);
    }
    if (lane < 16) part = fmaf(H2[r * LD2 + lane], __ldg(p.wout + 1 + kProj + lane), part);
    if (lane == 0) {
      const int G = p.n_genres;
      const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
      const int uid = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
      const int ig = genre_id(b.movie_genre, row, 3, G, b.err_flag);
      const int ug = genre_id(b.user_genre, row, 5, G, b.err_flag);
      float first = __fadd_rn(__ldg(p.blob + ly.first_cat_b), __ldg(p.blob + ly.first_num_b));
      if (ig >= 0) first += __ldg(p.first + ig);
      first += __ldg(p.first + G + mid);
      if (ug >= 0) first += __ldg(p.first + G + p.n_movies + ug);
      first += __ldg(p.first + (size_t)(2 * G + p.n_movies) + uid);
#pragma unroll
      for (int j = 0; j < kNumNumerics; ++j)
        first = fmaf(Xs[r * LDX + 4 * EP + j], __ldg(p.first_num + j), first);
      if (KEEP) firsts[r] = first;
      part = fmaf(first, __ldg(p.wout), part);
    }
    const float z = warp_sum(part) + __ldg(p.blob + ly.bout);
    if (lane == 0) emit(r, row, z);
  }
}

}  // namespace srs
