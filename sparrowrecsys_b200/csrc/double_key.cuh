// double_key.cuh - java.lang.Double.compare's order, descending, as an ascending unsigned key: every NaN is one
// key (0, first), then +inf .. +0.0, then -0.0 .. -inf.  binary_metrics.cu orders its thresholds by it and
// similar.cu its scores.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cstring>

namespace srs {

__device__ __forceinline__ uint64_t desc_key(double x) {
  if (x != x) return 0;
  uint64_t b;
  memcpy(&b, &x, 8);
  return (b >> 63) ? b : ~(b | (1ull << 63));
}
// the inverse of desc_key (NaN comes back as the canonical quiet NaN)
__device__ __forceinline__ double key_score(uint64_t k) {
  if (k == 0) return __longlong_as_double(0x7ff8000000000000ll);
  const uint64_t b = (k >> 63) ? k : ~k & ~(1ull << 63);
  return __longlong_as_double((long long)b);
}

}  // namespace srs
