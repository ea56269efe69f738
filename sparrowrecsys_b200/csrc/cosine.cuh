// cosine.cuh - Embedding.calculateSimilarity (online/model/Embedding.java:33-47) for one warp: float products
// accumulated in double, dot / (sqrt(n1) * sqrt(n2)).  util.cu's cosine_kernel (one query against n candidates)
// and similar.cu's emb ranker (each query against its genre candidates) share it; recforyou.cu's emb ranker takes
// the same sums one at a time (warp_product_sum).
#pragma once

#include <cuda_runtime.h>

namespace srs {

// The warp's three sums over q[0 .. dim) and v[0 .. dim): lane k takes elements k, k + 32, ..., then an xor tree;
// every lane ends with the totals.  All 32 lanes must call it.
__device__ __forceinline__ void cosine_sums(const float* __restrict__ q, const float* __restrict__ v, int dim,
                                            int lane, double& dot, double& n1, double& n2) {
  dot = 0.0, n1 = 0.0, n2 = 0.0;
  for (int k = lane; k < dim; k += 32) {
    const float a = __ldg(q + k), bb = __ldg(v + k);
    dot += (double)__fmul_rn(a, bb);
    n1 += (double)__fmul_rn(a, a);
    n2 += (double)__fmul_rn(bb, bb);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dot += __shfl_xor_sync(0xffffffffu, dot, o);
    n1 += __shfl_xor_sync(0xffffffffu, n1, o);
    n2 += __shfl_xor_sync(0xffffffffu, n2, o);
  }
}

// One of cosine_sums' three sums alone, sum of (double)(a[k] * b[k]): the same lane split and xor tree, so the same
// bits as the matching total of cosine_sums (a == b gives a squared norm).  recforyou.cu forms the norms once per
// call and only the dot per pair.  All 32 lanes must call it.
__device__ __forceinline__ double warp_product_sum(const float* __restrict__ a, const float* __restrict__ b, int dim,
                                                   int lane) {
  double s = 0.0;
  for (int k = lane; k < dim; k += 32) s += (double)__fmul_rn(__ldg(a + k), __ldg(b + k));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

__device__ __forceinline__ double cosine_value(double dot, double n1, double n2) {
  return dot / (sqrt(n1) * sqrt(n2));
}

}  // namespace srs
