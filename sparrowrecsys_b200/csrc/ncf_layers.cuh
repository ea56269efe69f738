// ncf_layers.cuh - the per-row Dense layers of NeuralCF, shared by the forward kernel (ncf.cu) and the
// training step (ncf_train.cu).  Weights are read from shared memory in the padded blob layout of NcfParams.
#pragma once

#include "common.cuh"

namespace srs {

template <int HP>
__device__ __forceinline__ void hidden_layer(float (&h)[HP], const float* __restrict__ W,
                                             const float* __restrict__ b) {
  float g[HP];
#pragma unroll
  for (int j = 0; j < HP; ++j) g[j] = b[j];
#pragma unroll
  for (int k = 0; k < HP; ++k) {
#pragma unroll
    for (int j = 0; j < HP; j += 4) {
      const float4 w = *reinterpret_cast<const float4*>(W + k * HP + j);
      g[j] = fmaf(h[k], w.x, g[j]);
      g[j + 1] = fmaf(h[k], w.y, g[j + 1]);
      g[j + 2] = fmaf(h[k], w.z, g[j + 2]);
      g[j + 3] = fmaf(h[k], w.w, g[j + 3]);
    }
  }
#pragma unroll
  for (int j = 0; j < HP; ++j) h[j] = fmaxf(g[j], 0.f);
}

// acc[j] += sum_{k<EP} row[k] * W[k][j]   (row streamed from global, W from smem)
template <int EP, int HP>
__device__ __forceinline__ void first_layer_accum(float (&acc)[HP], const float* __restrict__ row,
                                                  const float* __restrict__ W) {
  float4 v[EP / 4];
#pragma unroll
  for (int q = 0; q < EP / 4; ++q) v[q] = ldg4(row + 4 * q);
#pragma unroll
  for (int q = 0; q < EP / 4; ++q) {
    const float xs[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int j = 0; j < HP; j += 4) {
        const float4 w = *reinterpret_cast<const float4*>(W + (4 * q + kk) * HP + j);
        acc[j] = fmaf(xs[kk], w.x, acc[j]);
        acc[j + 1] = fmaf(xs[kk], w.y, acc[j + 1]);
        acc[j + 2] = fmaf(xs[kk], w.z, acc[j + 2]);
        acc[j + 3] = fmaf(xs[kk], w.w, acc[j + 3]);
      }
    }
  }
}

}  // namespace srs
