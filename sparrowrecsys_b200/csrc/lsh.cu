// lsh.cu - Spark ML's BucketedRandomProjectionLSH (the reference's embeddingLSH, Embedding.scala:230-252) on one
// device: the bucket ids of a set of vectors, and the single-probe approxNearestNeighbors of many keys at once.
// DESIGN.md section 4.14 gives the semantics; the unit vectors come from the host (embedding.py's `fit`).
//
//   lsh_hash_kernel   one thread per (row, table): floor(dot(x, v_j) / bucketLength), the dot sequential in double
//                     over the dimensions with each product and each sum rounded on its own (F2J ddot, no fma);
//   lsh_query_kernel  one block per key: the key's own bucket ids, then each warp scans a stride of the rows; a row
//                     sharing the key's bucket in at least one table is a candidate at distance sqrt(sum (x - key)^2)
//                     (sequential double), kept in the warp's sorted list of the best k under (distance, id, row)
//                     ascending; the eight lists are merged by one thread.  The best k under a strict total order do
//                     not depend on the order rows arrive in, so the result has one value.
#include <cuda_runtime.h>

#include <cmath>

#include "../../include/srs_ctr.h"
#include "hostcall.h"

namespace srs {
namespace {

constexpr int kMaxTables = 64;
constexpr int kMaxLshDim = 1024;
constexpr int kMaxK = 256;
constexpr int kQueryWarps = 8;
constexpr unsigned kFull = 0xffffffffu;

// BLAS.dot(x, v) / bucketLength, floored: F2J's ddot adds the products left to right from 0.0
template <class X>
__device__ __forceinline__ double bucket_of(const X* __restrict__ x, const double* __restrict__ v, int D, double bl) {
  double acc = 0.0;
  for (int d = 0; d < D; ++d) acc = __dadd_rn(acc, __dmul_rn((double)x[d], v[d]));
  return floor(__ddiv_rn(acc, bl));
}

__global__ void lsh_hash_kernel(const float* __restrict__ x, int64_t n, int D, const double* __restrict__ uv, int L,
                                double bl, double* __restrict__ out) {
  const int64_t nl = n * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / L;
    const int j = (int)(i - r * L);
    out[i] = bucket_of(x + r * D, uv + (int64_t)j * D, D, bl);
  }
}

struct Entry {
  double d;
  int32_t id, row;
};

__device__ __forceinline__ bool before(double d, int32_t id, int32_t row, const Entry& e) {
  return d < e.d || (d == e.d && (id < e.id || (id == e.id && row < e.row)));
}

// dynamic shared memory: kQueryWarps lists of k entries, then the key [D] and its bucket ids [L]
__global__ void __launch_bounds__(kQueryWarps * 32) lsh_query_kernel(
    const int32_t* __restrict__ ids, const float* __restrict__ x, const double* __restrict__ buckets, int n, int D,
    const double* __restrict__ uv, int L, double bl, const double* __restrict__ keys, int k,
    int32_t* __restrict__ out_ids, double* __restrict__ out_dist, int32_t* __restrict__ out_count) {
  extern __shared__ __align__(16) unsigned char smem[];
  Entry* lists = reinterpret_cast<Entry*>(smem);
  double* key = reinterpret_cast<double*>(lists + kQueryWarps * k);
  double* kh = key + D;
  __shared__ int sizes[kQueryWarps], head[kQueryWarps];
  const int q = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int d = threadIdx.x; d < D; d += blockDim.x) key[d] = keys[(int64_t)q * D + d];
  if (lane == 0) sizes[warp] = 0;
  __syncthreads();
  for (int j = threadIdx.x; j < L; j += blockDim.x) kh[j] = bucket_of(key, uv + (int64_t)j * D, D, bl);
  __syncthreads();

  Entry* list = lists + warp * k;
  int size = 0;
  for (int base = warp * 32; base < n; base += kQueryWarps * 32) {
    const int r = base + lane;
    bool cand = false;
    double dist = 0.0;
    int32_t id = 0;
    if (r < n) {
      const double* hb = buckets + (int64_t)r * L;
      for (int j = 0; j < L && !cand; ++j) cand = hb[j] == kh[j];
      if (cand) {
        const float* xr = x + (int64_t)r * D;
        double acc = 0.0;
        for (int d = 0; d < D; ++d) {
          const double diff = __dsub_rn((double)xr[d], key[d]);
          acc = __dadd_rn(acc, __dmul_rn(diff, diff));
        }
        dist = __dsqrt_rn(acc);
        id = ids[r];
      }
    }
    const bool want = cand && (size < k || before(dist, id, r, list[size - 1]));
    for (unsigned m = __ballot_sync(kFull, want); m; m &= m - 1) {
      const int src = __ffs(m) - 1;
      const double cd = __shfl_sync(kFull, dist, src);
      const int32_t cid = __shfl_sync(kFull, id, src);
      const int32_t crow = base + src;
      if (size == k && !before(cd, cid, crow, list[k - 1])) continue;   // an earlier lane raised the bar
      int pos = 0;                                       // entries that stay ahead of the new one
      for (int e0 = 0; e0 < size; e0 += 32) {
        const int e = e0 + lane;
        pos += __popc(__ballot_sync(kFull, e < size && !before(cd, cid, crow, list[e])));
      }
      const int last = size < k ? size : k - 1;          // entries [pos, last) move one place down, top 32 first
      for (int hi = last; hi > pos; hi -= 32) {
        const int e = hi - 1 - lane;
        Entry v;
        if (e >= pos) v = list[e];
        __syncwarp();
        if (e >= pos) list[e + 1] = v;
        __syncwarp();
      }
      if (lane == 0) list[pos] = Entry{cd, cid, crow};
      __syncwarp();
      if (size < k) ++size;
    }
  }
  if (lane == 0) sizes[warp] = size;
  __syncthreads();
  if (threadIdx.x == 0) {                                // merge the warps' sorted lists
    for (int w = 0; w < kQueryWarps; ++w) head[w] = 0;
    int c = 0;
    for (; c < k; ++c) {
      int best = -1;
      for (int w = 0; w < kQueryWarps; ++w) {
        if (head[w] == sizes[w]) continue;
        const Entry& e = lists[w * k + head[w]];
        if (best < 0 || before(e.d, e.id, e.row, lists[best * k + head[best]])) best = w;
      }
      if (best < 0) break;
      const Entry& e = lists[best * k + head[best]++];
      out_ids[(int64_t)q * k + c] = e.id;
      out_dist[(int64_t)q * k + c] = e.d;
    }
    out_count[q] = c;
  }
}

bool finite_f(const float* p, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (!std::isfinite(p[i])) return false;
  return true;
}

bool finite_d(const double* p, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (!std::isfinite(p[i])) return false;
  return true;
}

int check_model(const float* vectors, int64_t n, int32_t dim, const double* unit_vectors, int32_t num_tables,
                double bucket_length) {
  if (dim < 1 || dim > kMaxLshDim) return failf(SRS_ERR_INVALID, "dim %d outside 1..%d", dim, kMaxLshDim);
  if (num_tables < 1 || num_tables > kMaxTables)
    return failf(SRS_ERR_INVALID, "num_hash_tables %d outside 1..%d", num_tables, kMaxTables);
  if (!(bucket_length > 0) || !std::isfinite(bucket_length))
    return failf(SRS_ERR_INVALID, "bucket_length %g is not finite and > 0", bucket_length);
  if (n < 0 || n > INT32_MAX) return failf(SRS_ERR_INVALID, "n %lld outside 0..2^31-1", (long long)n);
  if (!unit_vectors || (n && !vectors)) return failf(SRS_ERR_INVALID, "null inputs");
  if (!finite_d(unit_vectors, (int64_t)num_tables * dim))
    return failf(SRS_ERR_INVALID, "a unit vector entry is not finite");
  if (!finite_f(vectors, n * dim)) return failf(SRS_ERR_INVALID, "a vector entry is not finite");
  return SRS_OK;
}

// the rows and unit vectors uploaded, and the rows' bucket ids [n][L] on the device
int hash_rows(HostCall& c, const float* vectors, int64_t n, int32_t dim, const double* unit_vectors, int32_t L,
              double bl, float** d_x, double** d_uv, double** d_buckets) {
  PROPAGATE(c.upload(d_x, vectors, n * dim));
  PROPAGATE(c.upload(d_uv, unit_vectors, (int64_t)L * dim));
  CUDA_TRY(c.sc.alloc(d_buckets, n * L));
  if (n) {
    const int T = 256;
    lsh_hash_kernel<<<grid_for(n * L, T), T, 0, c.s>>>(*d_x, n, dim, *d_uv, L, bl, *d_buckets);
    LAUNCHED();
  }
  return SRS_OK;
}

}  // namespace
}  // namespace srs

using namespace srs;

extern "C" int srs_lsh_transform_host(const float* vectors, int64_t n, int32_t dim, const double* unit_vectors,
                                      int32_t num_tables, double bucket_length, int32_t device, double* buckets) {
  PROPAGATE(check_model(vectors, n, dim, unit_vectors, num_tables, bucket_length));
  if (n && !buckets) return failf(SRS_ERR_INVALID, "null buckets");
  if (n == 0) return SRS_OK;
  HostCall c;
  PROPAGATE(c.begin(device));
  float* d_x;
  double *d_uv, *d_b;
  PROPAGATE(hash_rows(c, vectors, n, dim, unit_vectors, num_tables, bucket_length, &d_x, &d_uv, &d_b));
  CUDA_TRY(cudaMemcpyAsync(buckets, d_b, sizeof(double) * n * num_tables, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));
  return SRS_OK;
}

extern "C" int srs_lsh_query_host(const int32_t* ids, const float* vectors, int64_t n, int32_t dim,
                                  const double* unit_vectors, int32_t num_tables, double bucket_length,
                                  const double* keys, int32_t num_keys, int32_t k, int32_t device, int32_t* out_ids,
                                  double* out_dist, int32_t* out_count) {
  PROPAGATE(check_model(vectors, n, dim, unit_vectors, num_tables, bucket_length));
  if (n && !ids) return failf(SRS_ERR_INVALID, "null ids");
  if (k < 1 || k > kMaxK) return failf(SRS_ERR_INVALID, "k %d outside 1..%d", k, kMaxK);
  if (num_keys < 0) return failf(SRS_ERR_INVALID, "num_keys %d is negative", num_keys);
  if (num_keys && (!keys || !out_ids || !out_dist || !out_count))
    return failf(SRS_ERR_INVALID, "null keys or outputs");
  if (!finite_d(keys, (int64_t)num_keys * dim)) return failf(SRS_ERR_INVALID, "a key entry is not finite");
  if (num_keys == 0) return SRS_OK;
  HostCall c;
  PROPAGATE(c.begin(device));
  cudaStream_t s = c.s;
  float* d_x;
  double *d_uv, *d_b, *d_keys, *d_dist;
  int32_t *d_ids, *d_oid, *d_cnt;
  PROPAGATE(hash_rows(c, vectors, n, dim, unit_vectors, num_tables, bucket_length, &d_x, &d_uv, &d_b));
  PROPAGATE(c.upload(&d_ids, ids, n));
  PROPAGATE(c.upload(&d_keys, keys, (int64_t)num_keys * dim));
  CUDA_TRY(c.sc.alloc(&d_oid, (int64_t)num_keys * k)); CUDA_TRY(c.sc.alloc(&d_dist, (int64_t)num_keys * k));
  CUDA_TRY(c.sc.alloc(&d_cnt, num_keys));
  const size_t smem = sizeof(Entry) * kQueryWarps * k + sizeof(double) * (dim + num_tables);
  CUDA_TRY(cudaFuncSetAttribute(lsh_query_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  lsh_query_kernel<<<num_keys, kQueryWarps * 32, smem, s>>>(d_ids, d_x, d_b, (int)n, dim, d_uv, num_tables,
                                                             bucket_length, d_keys, k, d_oid, d_dist, d_cnt);
  LAUNCHED();
  CUDA_TRY(cudaMemcpyAsync(out_ids, d_oid, sizeof(int32_t) * num_keys * k, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out_dist, d_dist, sizeof(double) * num_keys * k, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out_count, d_cnt, sizeof(int32_t) * num_keys, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  return SRS_OK;
}
