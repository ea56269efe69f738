// lsh.cu - Spark ML's BucketedRandomProjectionLSH (the reference's embeddingLSH, Embedding.scala:230-252) on one
// device: the bucket ids of a set of vectors, the single-probe approxNearestNeighbors of many keys at once, and
// approxSimilarityJoin of two sets.  DESIGN.md section 4.14 gives the semantics; the unit vectors come from the host
// (embedding.py's `fit`).
//
//   lsh_hash_kernel   one thread per (row, table): floor(dot(x, v_j) / bucketLength), the dot sequential in double
//                     over the dimensions with each product and each sum rounded on its own (F2J ddot, no fma);
//   lsh_query_kernel  one block per key: the key's own bucket ids, then each warp scans a stride of the rows; a row
//                     sharing the key's bucket in at least one table is a candidate at distance sqrt(sum (x - key)^2)
//                     (sequential double), kept in the warp's sorted list of the best k under (distance, id, row)
//                     ascending; the eight lists are merged by one thread.  The best k under a strict total order do
//                     not depend on the order rows arrive in, so the result has one value.
//
// approxSimilarityJoin(A, B, threshold) - every (a, b) sharing a bucket in at least one table with distance <
// threshold, once - takes the tables one after another, so that a table's candidates (<= n_a * n_b < 2^62) index
// in int64 and no sum over tables is ever formed:
//   lsh_join_keys_kernel  B's bucket ids by table, -0.0 made +0.0 so that equal ids sort together;
//   per table j           a CUB radix sort of B's ids with their rows; lsh_join_runs_kernel gives each A row its
//                         run of equal ids (binary search); a CUB exclusive scan of the run lengths gives each A row
//                         its first candidate index and the table's C_j candidates;
//   lsh_join_kernel       cuts [0, C_j) into kJoinSegments contiguous segments, one block each, so that one huge
//                         bucket spreads over the whole GPU; a thread maps a candidate index to its A row (binary
//                         search of the offsets) and B row, and keeps the pair iff it collides in no earlier table
//                         (a pair belongs to the first table it collides in, which makes it distinct without a sort
//                         of candidates) and its distance is < threshold.  The counting pass writes each segment's
//                         count; after a CUB scan of all segments' counts and the capacity check, the fill pass
//                         walks the same segments and writes each kept pair at its segment's offset plus its rank in
//                         the block (a block scan per tile);
//   a CUB radix sort      of the P pairs by the 64-bit key (id_a, id_b), and lsh_join_ids_kernel splits the key.
// Scratch is O(L (n_a + n_b) + L kJoinSegments) plus the P-sized output: nothing grows with the candidate count.
// Positions come from scans over fixed segments and there are no atomics, so the same inputs give the same bits.
// Library kernel launches per join call with both sides non-empty (CUB's own are not counted):
//   3 + 2L        when P == 0 or P > capacity (the two hashes, the keys, per table the runs and the count);
//   4 + 3L        otherwise (plus per table the fill, and the id split).
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"

namespace srs {
namespace {

constexpr int kMaxTables = 64;
constexpr int kMaxLshDim = 1024;
constexpr int kMaxK = 256;
constexpr int kQueryWarps = 8;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kJoinThreads = 256;          // threads per join block: one tile of candidates
constexpr int kJoinSegments = 132 * 8;     // segments (blocks) per table in the join: eight per SM of the H100's 132

// BLAS.dot(x, v) / bucketLength, floored: F2J's ddot adds the products left to right from 0.0
template <class X>
__device__ __forceinline__ double bucket_of(const X* __restrict__ x, const double* __restrict__ v, int D, double bl) {
  double acc = 0.0;
  for (int d = 0; d < D; ++d) acc = __dadd_rn(acc, __dmul_rn((double)x[d], v[d]));
  return floor(__ddiv_rn(acc, bl));
}

// Vectors.sqdist's square root: sqrt(sum_d (x[d] - y[d])^2), both widened to double, summed left to right from 0.0
// with one rounding per operation.  (x - y)^2 == (y - x)^2 exactly, so the result is symmetric bit for bit.
template <class X, class Y>
__device__ __forceinline__ double distance(const X* __restrict__ x, const Y* __restrict__ y, int D) {
  double acc = 0.0;
  for (int d = 0; d < D; ++d) {
    const double diff = __dsub_rn((double)x[d], (double)y[d]);
    acc = __dadd_rn(acc, __dmul_rn(diff, diff));
  }
  return __dsqrt_rn(acc);
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
        dist = distance(x + (int64_t)r * D, key, D);
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

// B's bucket ids [n][L] by table: keys[j][r] = ids[r][j] + 0.0 (a floor of a tiny negative quotient is -0.0, equal
// to +0.0 but sorted apart from it); rows[r] = r
__global__ void lsh_join_keys_kernel(const double* __restrict__ buckets, int n, int L, double* __restrict__ keys,
                                     int32_t* __restrict__ rows) {
  const int64_t nl = (int64_t)n * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / L;
    const int j = (int)(i - r * L);
    keys[(int64_t)j * n + r] = __dadd_rn(buckets[i], 0.0);
    if (j == 0) rows[r] = (int32_t)r;
  }
}

// Table j's run of each A row among B's sorted ids: lo[r] = its first position, len[r] = its length; len[n_a] = 0, so
// that an exclusive scan of n_a + 1 lengths ends in the table's candidate count
__global__ void lsh_join_runs_kernel(const double* __restrict__ ba, int n_a, int L, int j,
                                     const double* __restrict__ skeys, int n_b, int32_t* __restrict__ lo,
                                     int64_t* __restrict__ len) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n_a; r += (int64_t)gridDim.x * blockDim.x) {
    if (r == n_a) {
      len[r] = 0;
      continue;
    }
    const double k = __dadd_rn(ba[r * L + j], 0.0);
    int a = 0, b = n_b;                                  // the first id >= k
    while (a < b) {
      const int m = a + ((b - a) >> 1);
      if (skeys[m] < k) a = m + 1; else b = m;
    }
    int e = a, f = n_b;                                  // the first id > k
    while (e < f) {
      const int m = e + ((f - e) >> 1);
      if (skeys[m] <= k) e = m + 1; else f = m;
    }
    lo[r] = a;
    len[r] = e - a;
  }
}

// The A row whose run holds candidate c: the largest r in [a, b] with off[r] <= c (a row with an empty run shares
// its offset with the next row, so the largest is the one whose run is not empty)
__device__ __forceinline__ int row_of(const int64_t* __restrict__ off, int a, int b, int64_t c) {
  while (a < b) {
    const int m = b - ((b - a) >> 1);
    if (off[m] <= c) a = m; else b = m - 1;
  }
  return a;
}

// (id_a, id_b) as one 64-bit key whose unsigned order is the pair's signed order
__device__ __forceinline__ unsigned long long pair_key(int32_t a, int32_t b) {
  return (unsigned long long)((uint32_t)a ^ 0x80000000u) << 32 | ((uint32_t)b ^ 0x80000000u);
}

// Table j's candidates: A row r with B rows rows[lo[r] ..) at indices off[r] .. off[r + 1) of [0, C_j), C_j =
// off[n_a].  Block g walks segment g of kJoinSegments contiguous ones in tiles of kJoinThreads.  A candidate is kept
// iff its buckets differ in every table before j and its distance is < threshold.  kFill false: seg[g] = the
// segment's kept count.  kFill true: seg[g] is the segment's first output position, and each kept pair is written
// there plus its rank in the segment, as pair_key and distance.
template <bool kFill>
__global__ void __launch_bounds__(kJoinThreads) lsh_join_kernel(
    const float* __restrict__ xa, const double* __restrict__ ba, int n_a, const float* __restrict__ xb,
    const double* __restrict__ bb, int D, int L, int j, const int64_t* __restrict__ off,
    const int32_t* __restrict__ lo, const int32_t* __restrict__ rows, double threshold,
    unsigned long long* __restrict__ seg, const int32_t* __restrict__ ids_a, const int32_t* __restrict__ ids_b,
    unsigned long long* __restrict__ out_key, double* __restrict__ out_dist) {
  using Scan = cub::BlockScan<int, kJoinThreads>;
  using Reduce = cub::BlockReduce<unsigned long long, kJoinThreads>;
  __shared__ union {
    typename Scan::TempStorage scan;
    typename Reduce::TempStorage reduce;
  } tmp;
  __shared__ int rows_of_segment[2];
  const int64_t C = off[n_a];
  const int64_t S = (C + kJoinSegments - 1) / kJoinSegments;
  const int64_t s0 = (int64_t)blockIdx.x * S;
  const int64_t s1 = s0 + S < C ? s0 + S : C;
  if (s0 >= s1) {
    if (!kFill && threadIdx.x == 0) seg[blockIdx.x] = 0;
    return;
  }
  if (threadIdx.x < 2) rows_of_segment[threadIdx.x] = row_of(off, 0, n_a - 1, threadIdx.x ? s1 - 1 : s0);
  __syncthreads();
  const int r0 = rows_of_segment[0], r1 = rows_of_segment[1];
  unsigned long long pos = kFill ? seg[blockIdx.x] : 0, kept = 0;
  for (int64_t t = s0; t < s1; t += kJoinThreads) {
    const int64_t c = t + threadIdx.x;
    bool keep = false;
    double dist = 0.0;
    int r = 0, b = 0;
    if (c < s1) {
      r = row_of(off, r0, r1, c);
      b = rows[lo[r] + (int)(c - off[r])];
      keep = true;
      for (int e = 0; e < j && keep; ++e) keep = ba[(int64_t)r * L + e] != bb[(int64_t)b * L + e];
      if (keep) {
        dist = distance(xa + (int64_t)r * D, xb + (int64_t)b * D, D);
        keep = dist < threshold;
      }
    }
    if (kFill) {
      if (__syncthreads_count(keep)) {                  // the same value in every thread
        int rank, total;
        Scan(tmp.scan).ExclusiveSum((int)keep, rank, total);
        if (keep) {
          out_key[pos + rank] = pair_key(ids_a[r], ids_b[b]);
          out_dist[pos + rank] = dist;
        }
        pos += total;
        __syncthreads();                                 // the next tile's scan reuses tmp
      }
    } else {
      kept += keep;
    }
  }
  if (!kFill) {
    const unsigned long long sum = Reduce(tmp.reduce).Sum(kept);
    if (threadIdx.x == 0) seg[blockIdx.x] = sum;
  }
}

// the sorted pair keys split into their ids
__global__ void lsh_join_ids_kernel(const unsigned long long* __restrict__ key, int64_t n, int32_t* __restrict__ ia,
                                    int32_t* __restrict__ ib) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    ia[i] = (int32_t)((uint32_t)(key[i] >> 32) ^ 0x80000000u);
    ib[i] = (int32_t)((uint32_t)key[i] ^ 0x80000000u);
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

// ids of one side of a join: non-null when n > 0, and no id twice
int check_join_ids(const int32_t* ids, int64_t n, const char* side) {
  if (n && !ids) return failf(SRS_ERR_INVALID, "null ids_%s", side);
  std::vector<int32_t> v(ids, ids + n);
  std::sort(v.begin(), v.end());
  const auto dup = std::adjacent_find(v.begin(), v.end());
  if (dup != v.end()) return failf(SRS_ERR_INVALID, "ids_%s holds id %d more than once", side, (int)*dup);
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

extern "C" int srs_lsh_similarity_join_host(const int32_t* ids_a, const float* vectors_a, int64_t n_a,
                                            const int32_t* ids_b, const float* vectors_b, int64_t n_b, int32_t dim,
                                            const double* unit_vectors, int32_t num_tables, double bucket_length,
                                            double threshold, int32_t device, int64_t capacity, int32_t* out_ids_a,
                                            int32_t* out_ids_b, double* out_dist, int64_t* n_pairs) {
  PROPAGATE(check_model(vectors_a, n_a, dim, unit_vectors, num_tables, bucket_length));
  PROPAGATE(check_model(vectors_b, n_b, dim, unit_vectors, num_tables, bucket_length));
  PROPAGATE(check_join_ids(ids_a, n_a, "a"));
  PROPAGATE(check_join_ids(ids_b, n_b, "b"));
  if (capacity < 0) return failf(SRS_ERR_INVALID, "capacity %lld is negative", (long long)capacity);
  if (!n_pairs) return failf(SRS_ERR_INVALID, "null n_pairs");
  if (capacity > 0 && (!out_ids_a || !out_ids_b || !out_dist)) return failf(SRS_ERR_INVALID, "null outputs");
  if (n_a == 0 || n_b == 0) {
    *n_pairs = 0;
    return SRS_OK;
  }
  HostCall c;
  PROPAGATE(c.begin(device));
  cudaStream_t s = c.s;
  const int na = (int)n_a, nb = (int)n_b, L = num_tables, G = kJoinSegments, T = kJoinThreads;
  float *d_xa, *d_xb;
  double *d_uva, *d_uvb, *d_ba, *d_bb, *d_keys, *d_skeys;
  int32_t *d_ida, *d_idb, *d_iota, *d_rows, *d_lo;
  int64_t *d_len, *d_off;
  unsigned long long *d_cnt, *d_base;
  PROPAGATE(hash_rows(c, vectors_a, n_a, dim, unit_vectors, L, bucket_length, &d_xa, &d_uva, &d_ba));
  PROPAGATE(hash_rows(c, vectors_b, n_b, dim, unit_vectors, L, bucket_length, &d_xb, &d_uvb, &d_bb));
  PROPAGATE(c.upload(&d_ida, ids_a, n_a));
  PROPAGATE(c.upload(&d_idb, ids_b, n_b));
  CUDA_TRY(c.sc.alloc(&d_keys, (int64_t)L * nb)); CUDA_TRY(c.sc.alloc(&d_skeys, nb));
  CUDA_TRY(c.sc.alloc(&d_iota, nb)); CUDA_TRY(c.sc.alloc(&d_rows, (int64_t)L * nb));
  CUDA_TRY(c.sc.alloc(&d_lo, (int64_t)L * na)); CUDA_TRY(c.sc.alloc(&d_len, n_a + 1));
  CUDA_TRY(c.sc.alloc(&d_off, (int64_t)L * (n_a + 1)));
  CUDA_TRY(c.sc.alloc(&d_cnt, (int64_t)L * G + 1)); CUDA_TRY(c.sc.alloc(&d_base, (int64_t)L * G + 1));
  CUDA_TRY(cudaMemsetAsync(d_cnt, 0, sizeof(unsigned long long) * ((int64_t)L * G + 1), s));
  lsh_join_keys_kernel<<<grid_for(n_b * L, T), T, 0, s>>>(d_bb, nb, L, d_keys, d_iota);
  LAUNCHED();
  for (int j = 0; j < L; ++j) {                          // the counting pass, one table after another
    int32_t* rows = d_rows + (int64_t)j * nb;
    int32_t* lo = d_lo + (int64_t)j * na;
    int64_t* off = d_off + (int64_t)j * (n_a + 1);
    CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_keys + (int64_t)j * nb, d_skeys, d_iota, rows, nb,
                                               0, 64, s));
    lsh_join_runs_kernel<<<grid_for(n_a + 1, T), T, 0, s>>>(d_ba, na, L, j, d_skeys, nb, lo, d_len);
    LAUNCHED();
    CUB_RUN(c, cub::DeviceScan::ExclusiveSum(tmp__, tb__, d_len, off, na + 1, s));
    lsh_join_kernel<false><<<G, T, 0, s>>>(d_xa, d_ba, na, d_xb, d_bb, dim, L, j, off, lo, rows, threshold,
                                           d_cnt + (int64_t)j * G, d_ida, d_idb, nullptr, nullptr);
    LAUNCHED();
  }
  CUB_RUN(c, cub::DeviceScan::ExclusiveSum(tmp__, tb__, d_cnt, d_base, L * G + 1, s));
  unsigned long long P = 0;
  CUDA_TRY(cudaMemcpyAsync(&P, d_base + (int64_t)L * G, sizeof(P), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  *n_pairs = (int64_t)P;
  if ((int64_t)P > capacity)
    return failf(SRS_ERR_RANGE, "the join has %lld pairs, more than the capacity %lld", (long long)P,
                 (long long)capacity);
  if (P == 0) return SRS_OK;
  unsigned long long *d_key, *d_skey;
  double *d_dist, *d_sdist;
  int32_t *d_oa, *d_ob;
  CUDA_TRY(c.sc.alloc(&d_key, P)); CUDA_TRY(c.sc.alloc(&d_skey, P));
  CUDA_TRY(c.sc.alloc(&d_dist, P)); CUDA_TRY(c.sc.alloc(&d_sdist, P));
  CUDA_TRY(c.sc.alloc(&d_oa, P)); CUDA_TRY(c.sc.alloc(&d_ob, P));
  for (int j = 0; j < L; ++j) {                          // the fill pass: the same walk, writing
    lsh_join_kernel<true><<<G, T, 0, s>>>(d_xa, d_ba, na, d_xb, d_bb, dim, L, j, d_off + (int64_t)j * (n_a + 1),
                                          d_lo + (int64_t)j * na, d_rows + (int64_t)j * nb, threshold,
                                          d_base + (int64_t)j * G, d_ida, d_idb, d_key, d_dist);
    LAUNCHED();
  }
  CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_key, d_skey, d_dist, d_sdist, (int64_t)P, 0, 64, s));
  lsh_join_ids_kernel<<<grid_for((int64_t)P, T), T, 0, s>>>(d_skey, (int64_t)P, d_oa, d_ob);
  LAUNCHED();
  CUDA_TRY(cudaMemcpyAsync(out_ids_a, d_oa, sizeof(int32_t) * P, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out_ids_b, d_ob, sizeof(int32_t) * P, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out_dist, d_sdist, sizeof(double) * P, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  return SRS_OK;
}
