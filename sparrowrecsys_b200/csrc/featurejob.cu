// featurejob.cu - the reference's FeatureEngineering job (OFF/featureeng/FeatureEngineering.scala) and the sample /
// split tail of FeatureEngForRecModel (:176-205) on one device.  DESIGN.md section 4.16 gives the semantics.
//
//   approxQuantile       values -> order-preserving 64-bit keys -> CUB radix sort -> fj_compress_kernel (one
//                        thread: Spark's compressImmut walk over the sorted samples, jumping over each merged run)
//                        -> fj_query_kernel (one thread per probability: the query's minRank / maxRank walk);
//   QuantileDiscretizer  the quantiles at i / N, fj_splits_kernel (ends to -inf / +inf, order-keeping distinct,
//                        strictly increasing check) and fj_bucket_kernel (Bucketizer's binary search);
//   MinMaxScaler         CUB min / max over the keys, fj_scale_kernel;
//   rating features      featureeng.cu's integer moment kernel, DeviceSelect of the rated movies, fj_rating_kernel;
//   StringIndexer        integer-atomic word histogram, one radix sort by (descending count, Scala 2.11 hash-trie
//                        order), then for the multi-hot vectors a radix sort of the movies and a CSR assembly;
//   sample / split       fj_part_kernel (counter-based uniforms) and one DeviceSelect per part.
// No float atomics: every run gives the same bits.  Every host entry checks its inputs before any launch.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <charconv>
#include <cmath>
#include <cstdio>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"

namespace srs {
namespace {

constexpr int64_t kMaxValues = 2147483647;      // int32 row indices
constexpr int kMaxProbs = 1 << 16;
constexpr int kMaxBuckets = 10000;
constexpr int kMaxWords = 1 << 20;
constexpr int64_t kMaxTokens = (1 << 29) - 1;   // the count field of a label's sort key
constexpr int kMaxWordsPerRow = 256;
constexpr int kMaxParts = 64;
constexpr int32_t kMaxMovieId = (1 << 24) - 1;
constexpr int64_t kMaxRatings = 21000000;       // featureeng.cu's bound: every Q and 4n(n-1) below 2^53

// a grid-stride loop over 0..n-1 with a 64-bit index: n may come within one grid stride of INT32_MAX
#define FJ_GRID_STRIDE(i, n) \
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// java.lang.Double.compare's total order (-0.0 < 0.0) as unsigned keys; no key of a non-NaN value is ~0
__host__ __device__ __forceinline__ uint64_t order_key(double x) {
  uint64_t b;
  memcpy(&b, &x, 8);
  return (b >> 63) ? ~b : (b | (1ull << 63));
}
__host__ __device__ __forceinline__ double key_value(uint64_t k) {
  const uint64_t b = (k >> 63) ? (k & ~(1ull << 63)) : ~k;
  double x;
  memcpy(&x, &b, 8);
  return x;
}

// scala.collection.immutable.HashMap.improve (2.11)
__host__ __device__ __forceinline__ uint32_t improve(int32_t hcode) {
  uint32_t h = (uint32_t)hcode;
  h = h + ~(h << 9);
  h = h ^ (h >> 14);
  h = h + (h << 4);
  return h ^ (h >> 10);
}

// the hash trie's iteration order: improve(hashCode) as 5-bit digits from the low bits, lowest digit first (35 bits)
__host__ __device__ __forceinline__ uint64_t trie_key(int32_t hcode) {
  const uint32_t h = improve(hcode);
  uint64_t k = 0;
  for (int level = 0; level < 7; ++level) k = (k << 5) | ((h >> (5 * level)) & 31u);
  return k;
}

__global__ void fj_keys_kernel(const double* __restrict__ v, int n, uint64_t* __restrict__ keys) {
  FJ_GRID_STRIDE(i, n) keys[i] = order_key(v[i]);
}

// QuantileSummaries with every value in one head buffer: withHeadBufferInserted gives sample j (sorted) g = 1 and
// delta = floor(2 eps (j + 1)), 0 at both ends; compressImmut (mergeThreshold T = 2 eps n) walks from the top: a
// head with delta d absorbs the samples below it while 1 + g + d < T, i.e. t = ceil(T - 2 - d) of them (at most
// down to sample 1), so the next head is t + 1 lower.  Delta is constant over runs of sorted indices, and so is t:
// within a run the heads are an arithmetic progression.  The walk therefore takes one step per run (a segment:
// top head, stride, count) or per head, whichever comes first - at most min(heads, runs + 3) steps, runs <= 2 eps
// n + 1 - and fj_expand_kernel writes the heads in parallel.
struct QSegment {
  long long top, stride, count, start;   // heads top, top - stride, ...; `start` heads precede it in walk order
  long long g, d;
};

__device__ __forceinline__ long long qs_delta(long long j, long long n, double e2) {
  return (j == 0 || j == n - 1) ? 0 : (long long)floor(e2 * (double)(j + 1));
}

__global__ void fj_compress_kernel(const int* __restrict__ d_n, double eps, QSegment* __restrict__ seg, int seg_cap,
                                   int* __restrict__ n_seg, long long* __restrict__ m_out, int* __restrict__ err) {
  const long long n = *d_n;
  *err = 0;
  if (n <= 0) { *n_seg = 0; *m_out = 0; return; }
  const double e2 = 2.0 * eps;
  const double T = e2 * (double)n;
  int ns = 0;
  long long heads = 0, j = n - 1;
  for (;;) {
    const long long d = qs_delta(j, n, e2);
    const double x = T - (double)(d + 2);
    const long long t = x > 0.0 ? (long long)ceil(x) : 0;    // unclamped
    QSegment sg;
    sg.top = j;
    sg.d = d;
    sg.start = heads;
    if (j >= 1 && j <= n - 2 && t <= j - 1) {
      long long a = 1, b = j;                                 // the run of d starts at the least a with delta >= d
      while (a < b) {
        const long long mid = (a + b) >> 1;
        if (qs_delta(mid, n, e2) >= d) b = mid; else a = mid + 1;
      }
      const long long lo = a > t + 1 ? a : t + 1;            // below t + 1 the take would be clamped
      sg.stride = t + 1;
      sg.count = (j - lo) / (t + 1) + 1;
      sg.g = 1 + t;
    } else {
      const long long take = t < (j >= 1 ? j - 1 : 0) ? t : (j >= 1 ? j - 1 : 0);
      sg.stride = take + 1;
      sg.count = 1;
      sg.g = 1 + take;
    }
    if (ns == seg_cap) { *err = 1; return; }
    seg[ns++] = sg;
    heads += sg.count;
    j -= sg.count * sg.stride;
    if (j < 1) break;
  }
  *n_seg = ns;
  *m_out = heads + (n > 1);                                 // the minimum is kept apart
}

// the samples in ascending order: s[0] is the minimum (when n > 1), s[m - 1] the top head
__global__ void fj_expand_kernel(const QSegment* __restrict__ seg, const int* __restrict__ n_seg,
                                 const long long* __restrict__ d_m, const int* __restrict__ d_n,
                                 int32_t* __restrict__ s_idx, long long* __restrict__ s_g, long long* __restrict__ s_d) {
  const long long m = *d_m, n = *d_n;
  const int ns = *n_seg;
  const long long heads = m - (n > 1);
  FJ_GRID_STRIDE(p, heads) {
    int a = 0, b = ns - 1;                                  // the last segment with start <= p
    while (a < b) {
      const int mid = (a + b + 1) >> 1;
      if (seg[mid].start <= p) a = mid; else b = mid - 1;
    }
    const QSegment& sg = seg[a];
    const long long at = m - 1 - p;
    s_idx[at] = (int32_t)(sg.top - sg.stride * (p - sg.start));
    s_g[at] = sg.g;
    s_d[at] = sg.d;
    if (p == 0 && n > 1) { s_idx[0] = 0; s_g[0] = 1; s_d[0] = 0; }
  }
}

// QuantileSummaries.query: p <= eps -> the minimum, p >= 1 - eps -> the maximum; otherwise the first sample (all
// but the last) with maxRank - targetError <= rank <= minRank + targetError, rank = ceil(p n), targetError =
// ceil(eps n); none -> the last.  minRank (the prefix sums of g) increases strictly and delta does not decrease
// below the last sample, so the right-hand test holds on a suffix and the left-hand one on a prefix: the answer is
// the first sample passing the right-hand test if it also passes the left-hand one.  A binary search.  NaN when
// there are no values.
__global__ void fj_query_kernel(const uint64_t* __restrict__ sorted, const int* __restrict__ d_n,
                                const int32_t* __restrict__ s_idx, const long long* __restrict__ s_minr,
                                const long long* __restrict__ s_d, const long long* __restrict__ d_m,
                                const double* __restrict__ probs, int np, double eps, double* __restrict__ out) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= np) return;
  const long long m = *d_m, n = *d_n;
  if (m == 0) { out[q] = __longlong_as_double(0x7ff8000000000000ll); return; }
  const double p = probs[q];
  long long pick = m - 1;
  if (p <= eps) {
    pick = 0;
  } else if (p < 1.0 - eps) {
    const double rank = (double)(long long)ceil(p * (double)n);
    const double te = ceil(eps * (double)n);
    long long a = 0, b = m - 1;                             // the first a < m - 1 with rank <= minRank + te
    while (a < b) {
      const long long mid = (a + b) >> 1;
      if (rank <= (double)s_minr[mid] + te) b = mid; else a = mid + 1;
    }
    if (a < m - 1 && (double)(s_minr[a] + s_d[a]) - te <= rank) pick = a;
  }
  out[q] = key_value(sorted[s_idx[pick]]);
}

// QuantileDiscretizer.fit's tail: the ends become -inf / +inf, then `distinct` (bit equality, first occurrence
// kept); the Bucketizer needs >= 3 strictly increasing splits, else *err = 1.  One block.
__global__ void fj_splits_kernel(const double* __restrict__ q, int nq, double* __restrict__ splits,
                                 int* __restrict__ n_splits, int* __restrict__ err, uint8_t* __restrict__ dup) {
  auto at = [&](int k) {
    return k == 0 ? -INFINITY : k == nq - 1 ? INFINITY : q[k];
  };
  for (int k = threadIdx.x; k < nq; k += blockDim.x) {
    const long long bk = __double_as_longlong(at(k));
    uint8_t d = 0;
    for (int j = 0; j < k && !d; ++j) d = __double_as_longlong(at(j)) == bk;
    dup[k] = d;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int c = 0, bad = 0;
    for (int k = 0; k < nq; ++k) {
      if (dup[k]) continue;
      const double v = at(k);
      if (c && !(splits[c - 1] < v)) bad = 1;
      splits[c++] = v;
    }
    *n_splits = c;
    *err = bad || c < 3;
  }
}

// Bucketizer: a value equal to the last split -> the last bucket; otherwise Arrays.binarySearch in Double's total
// order: the index of the last split <= x (a value on a split goes to the bucket above it)
__global__ void fj_bucket_kernel(const double* __restrict__ v, int n, const double* __restrict__ splits,
                                 const int* __restrict__ d_ns, int32_t* __restrict__ out) {
  const int ns = *d_ns;
  FJ_GRID_STRIDE(i, n) {
    const double x = v[i];
    if (x == splits[ns - 1]) { out[i] = ns - 2; continue; }
    const uint64_t k = order_key(x);
    int lo = 0, hi = ns;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (order_key(splits[mid]) > k) hi = mid; else lo = mid + 1;
    }
    out[i] = lo - 1;
  }
}

// MinMaxScalerModel.transform with min 0, max 1: ((x - Emin) / (Emax - Emin)) * 1 + 0, or 0.5 * 1 + 0 for a zero
// range; each operation rounded once
__global__ void fj_scale_kernel(const double* __restrict__ v, int n, const uint64_t* __restrict__ kmin,
                                const uint64_t* __restrict__ kmax, double* __restrict__ out) {
  const double lo = key_value(*kmin), hi = key_value(*kmax);
  const double range = __dsub_rn(hi, lo);
  FJ_GRID_STRIDE(i, n) {
    const double raw = range != 0.0 ? __ddiv_rn(__dsub_rn(v[i], lo), range) : 0.5;
    out[i] = __dadd_rn(__dmul_rn(raw, 1.0), 0.0);
  }
}

__global__ void fj_rated_kernel(const unsigned long long* __restrict__ mmom, int slots, int32_t* __restrict__ iota,
                                uint8_t* __restrict__ flag) {
  FJ_GRID_STRIDE(m, slots) {
    iota[m] = m;
    flag[m] = mmom[3 * (size_t)m] != 0;
  }
}

// groupBy(movieId).agg(count, avg, variance): avg = S1 / (2n), var_samp = Q / (4n(n - 1)), Q = n S2 - S1^2 (half-
// stars), each one correctly rounded division of integers below 2^53; a null variance (n = 1) is NaN
__global__ void fj_rating_kernel(const unsigned long long* __restrict__ mmom, const int32_t* __restrict__ ids,
                                 const int* __restrict__ d_count, int64_t* __restrict__ cnt, double* __restrict__ avg,
                                 double* __restrict__ var) {
  const int total = *d_count;
  FJ_GRID_STRIDE(k, total) {
    const size_t m = (size_t)ids[k];
    const long long n = (long long)mmom[3 * m], s1 = (long long)mmom[3 * m + 1], s2 = (long long)mmom[3 * m + 2];
    cnt[k] = n;
    avg[k] = __ddiv_rn((double)s1 * 0.5, (double)n);
    var[k] = n >= 2 ? __ddiv_rn((double)(n * s2 - s1 * s1), (double)(4 * n * (n - 1)))
                    : __longlong_as_double(0x7ff8000000000000ll);
  }
}

__global__ void fj_hist_kernel(const int32_t* __restrict__ tok, int n, unsigned long long* __restrict__ cnt) {
  FJ_GRID_STRIDE(i, n) atomicAdd(cnt + tok[i], 1ull);
}

// a word's label sort key: descending count, then the hash trie's iteration order (countByValue's map; sortBy is
// stable)
__global__ void fj_label_key_kernel(const unsigned long long* __restrict__ cnt, const int32_t* __restrict__ hash,
                                    int W, uint64_t* __restrict__ key, int32_t* __restrict__ word) {
  FJ_GRID_STRIDE(w, W) {
    key[w] = ((uint64_t)(kMaxTokens - (int64_t)cnt[w]) << 35) | trie_key(hash[w]);
    word[w] = w;
  }
}

__global__ void fj_label_index_kernel(const int32_t* __restrict__ sorted_word, const unsigned long long* __restrict__ cnt,
                                      int W, int32_t* __restrict__ label_of, int64_t* __restrict__ label_cnt) {
  FJ_GRID_STRIDE(k, W) {
    const int w = sorted_word[k];
    label_of[w] = k;
    label_cnt[k] = (int64_t)cnt[w];
  }
}

__global__ void fj_row_iota_kernel(const int32_t* __restrict__ movie, int n, uint32_t* __restrict__ key,
                                   int32_t* __restrict__ iota) {
  FJ_GRID_STRIDE(i, n) {
    key[i] = (uint32_t)movie[i];
    iota[i] = i;
  }
}

__global__ void fj_row_len_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ off, int n,
                                  int32_t* __restrict__ len) {
  FJ_GRID_STRIDE(r, n) {
    const int src = order[r];
    len[r] = off[src + 1] - off[src];
  }
}

// the multi-hot vector of output row r: its words' label indices, sorted ascending (array2vec's sortWith(_ < _))
__global__ void fj_csr_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ off,
                              const int32_t* __restrict__ tok, const int32_t* __restrict__ label_of, int n,
                              const int32_t* __restrict__ out_off, int32_t* __restrict__ out_idx) {
  FJ_GRID_STRIDE(r, n) {
    const int src = order[r];
    const int b = off[src], len = off[src + 1] - b;
    int32_t* dst = out_idx + out_off[r];
    for (int p = 0; p < len; ++p) {
      const int v = label_of[tok[b + p]];
      int q = p;
      while (q > 0 && dst[q - 1] > v) { dst[q] = dst[q - 1]; --q; }
      dst[q] = v;
    }
  }
}

struct Bounds {
  double b[kMaxParts + 1];
};

// part of row i: -1 when not sampled (stream-0 uniform >= fraction); else the j with lb_j <= u < ub_j for its
// stream-1 uniform (-1 if none: the bounds' rounding can leave a gap below 1)
__global__ void fj_part_kernel(int n, uint64_t key0, uint64_t key1, double fraction, Bounds bounds, int n_parts,
                               int8_t* __restrict__ part) {
  FJ_GRID_STRIDE(i, n) {
    int8_t p = -1;
    if (uniform53(key0, (uint64_t)i) < fraction) {
      const double u = uniform53(key1, (uint64_t)i);
      for (int j = 0; j < n_parts; ++j)
        if (u >= bounds.b[j] && u < bounds.b[j + 1]) { p = (int8_t)j; break; }
    }
    part[i] = p;
  }
}

// the sampled rows' timestamps as sort keys (unsampled rows: ~0, after every value); sampled flags
__global__ void fj_ts_keys_kernel(const int64_t* __restrict__ ts, int n, uint64_t key0, double fraction,
                                  uint64_t* __restrict__ keys, uint8_t* __restrict__ flag) {
  FJ_GRID_STRIDE(i, n) {
    const bool s = uniform53(key0, (uint64_t)i) < fraction;
    keys[i] = s ? order_key((double)ts[i]) : ~0ull;
    flag[i] = s;
  }
}

// timestampLong <= splitTimestamp (the long compared as a double) -> training (0), else test (1)
__global__ void fj_ts_part_kernel(const int64_t* __restrict__ ts, const uint8_t* __restrict__ flag, int n,
                                  const double* __restrict__ split, int8_t* __restrict__ part) {
  const double t = *split;
  FJ_GRID_STRIDE(i, n)
    part[i] = flag[i] ? ((double)ts[i] <= t ? 0 : 1) : -1;
}

// the radix-sort keys of gather_parts (part -1 -> 255, after every part), the row indices, and each part's count:
// per-block shared counters, then one integer atomic per block and part (order-free)
__global__ void fj_part_count_kernel(const int8_t* __restrict__ part, int n, int n_parts, uint8_t* __restrict__ key,
                                     int32_t* __restrict__ iota, unsigned long long* __restrict__ cnt) {
  __shared__ unsigned int c[kMaxParts];
  for (int j = threadIdx.x; j < n_parts; j += blockDim.x) c[j] = 0;
  __syncthreads();
  FJ_GRID_STRIDE(i, n) {
    const int p = part[i];
    key[i] = (uint8_t)p;
    iota[i] = (int32_t)i;
    if (p >= 0) atomicAdd(&c[p], 1u);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < n_parts; j += blockDim.x)
    if (c[j]) atomicAdd(cnt + j, (unsigned long long)c[j]);
}

// the number of set flags: a block count, then one integer atomic per block
__global__ void fj_flag_count_kernel(const uint8_t* __restrict__ flag, int n, int* __restrict__ count) {
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < n; base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const int c = __syncthreads_count(i < n && flag[i]);
    if (threadIdx.x == 0 && c) atomicAdd(count, c);
  }
}

// ------------------------------------------------------------------------------------------------- host side
// approxQuantile of the first *d_n of n_cap device keys (sorted in place) at np device probabilities -> d_out
int quantiles_of_keys(HostCall& r, uint64_t* d_keys, int n_cap, const int* d_n, const double* d_probs, int np,
                      double eps, double* d_out) {
  // segments: at most min(heads, runs + 3), runs <= 2 eps n + 1 (fj_compress_kernel)
  const long long by_runs = (long long)(2.0 * eps * (double)n_cap) + 8;
  const int seg_cap = (int)std::min<long long>(n_cap, by_runs) + 2;
  uint64_t* d_sorted;
  int32_t* s_idx;
  long long *s_g, *s_minr, *s_d, *d_m;
  QSegment* d_seg;
  int *d_nseg, *d_err;
  CUDA_TRY(r.sc.alloc(&d_sorted, n_cap));
  CUDA_TRY(r.sc.alloc(&s_idx, n_cap));
  CUDA_TRY(r.sc.alloc(&s_g, n_cap));
  CUDA_TRY(r.sc.alloc(&s_minr, n_cap));
  CUDA_TRY(r.sc.alloc(&s_d, n_cap));
  CUDA_TRY(r.sc.alloc(&d_m, 1));
  CUDA_TRY(r.sc.alloc(&d_seg, seg_cap));
  CUDA_TRY(r.sc.alloc(&d_nseg, 1));
  CUDA_TRY(r.sc.alloc(&d_err, 1));
  CUB_RUN(r, cub::DeviceRadixSort::SortKeys(tmp__, tb__, d_keys, d_sorted, n_cap, 0, 64, r.s));
  fj_compress_kernel<<<1, 1, 0, r.s>>>(d_n, eps, d_seg, seg_cap, d_nseg, d_m, d_err);
  LAUNCHED();
  fj_expand_kernel<<<grid_for(n_cap, 256), 256, 0, r.s>>>(d_seg, d_nseg, d_m, d_n, s_idx, s_g, s_d);
  LAUNCHED();
  // entries past m are never read: the prefix sums below m do not depend on them
  CUB_RUN(r, cub::DeviceScan::InclusiveSum(tmp__, tb__, s_g, s_minr, n_cap, r.s));
  fj_query_kernel<<<(np + 127) / 128, 128, 0, r.s>>>(d_sorted, d_n, s_idx, s_minr, s_d, d_m, d_probs, np, eps, d_out);
  LAUNCHED();
  int err = 0;
  CUDA_TRY(cudaMemcpyAsync(&err, d_err, sizeof(int), cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  if (err) return failf(SRS_ERR_INVALID, "approxQuantile: more compress segments than the bound %d", seg_cap);
  return SRS_OK;
}

int check_values(const double* v, int64_t n, const char* what) {
  if (n < 1 || n > kMaxValues) return failf(SRS_ERR_INVALID, "%s: n %lld outside 1..%lld", what, (long long)n,
                                              (long long)kMaxValues);
  if (!v) return failf(SRS_ERR_INVALID, "%s: null values", what);
  for (int64_t i = 0; i < n; ++i)
    if (std::isnan(v[i])) return failf(SRS_ERR_INVALID, "%s: value %lld is NaN", what, (long long)i);
  return SRS_OK;
}

int check_eps(double eps) {
  if (!(eps >= 0.0 && eps <= 1.0)) return failf(SRS_ERR_INVALID, "relative_error %g outside [0, 1]", eps);
  return SRS_OK;
}

// device values -> keys, then the quantiles at host probabilities into d_out
int quantiles_of_values(HostCall& r, const double* d_v, int n, const double* probs, int np, double eps, double* d_out) {
  uint64_t* d_keys;
  double* d_probs;
  int* d_n;
  CUDA_TRY(r.sc.alloc(&d_keys, n));
  PROPAGATE(r.upload(&d_probs, probs, np));
  PROPAGATE(r.upload(&d_n, &n, 1));
  fj_keys_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_v, n, d_keys);
  LAUNCHED();
  return quantiles_of_keys(r, d_keys, n, d_n, d_probs, np, eps, d_out);
}

int check_splits(const double* splits, int32_t n_splits) {
  if (!splits || n_splits < 3 || n_splits > kMaxBuckets + 1)
    return failf(SRS_ERR_INVALID, "splits: need 3..%d values", kMaxBuckets + 1);
  for (int k = 0; k < n_splits; ++k) {
    if (std::isnan(splits[k])) return failf(SRS_ERR_INVALID, "split %d is NaN", k);
    if (k && !(splits[k - 1] < splits[k])) return failf(SRS_ERR_INVALID, "splits must be strictly increasing");
  }
  return SRS_OK;
}

// the word-histogram and label order shared by the StringIndexer and the multi-hot encoder; d_label_of [W] and
// d_label_word / d_label_cnt [W] on the device
int index_labels(HostCall& r, const int32_t* d_tok, int n_tok, const int32_t* hash, int W, int32_t** d_label_of,
                 int32_t** d_label_word, int64_t** d_label_cnt) {
  unsigned long long* d_cnt;
  int32_t *d_hash, *d_word;
  uint64_t *d_key, *d_key2;
  CUDA_TRY(r.sc.alloc(&d_cnt, W));
  PROPAGATE(r.upload(&d_hash, hash, W));
  CUDA_TRY(r.sc.alloc(&d_word, W));
  CUDA_TRY(r.sc.alloc(&d_key, W));
  CUDA_TRY(r.sc.alloc(&d_key2, W));
  CUDA_TRY(r.sc.alloc(d_label_of, W));
  CUDA_TRY(r.sc.alloc(d_label_word, W));
  CUDA_TRY(r.sc.alloc(d_label_cnt, W));
  CUDA_TRY(cudaMemsetAsync(d_cnt, 0, sizeof(unsigned long long) * W, r.s));
  fj_hist_kernel<<<grid_for(n_tok, 256), 256, 0, r.s>>>(d_tok, n_tok, d_cnt);
  LAUNCHED();
  fj_label_key_kernel<<<grid_for(W, 256), 256, 0, r.s>>>(d_cnt, d_hash, W, d_key, d_word);
  LAUNCHED();
  CUB_RUN(r, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_key, d_key2, d_word, *d_label_word, W, 0, 64, r.s));
  fj_label_index_kernel<<<grid_for(W, 256), 256, 0, r.s>>>(*d_label_word, d_cnt, W, *d_label_of, *d_label_cnt);
  LAUNCHED();
  return SRS_OK;
}

int check_tokens(const int32_t* tok, int64_t n_tok, const int32_t* hash, int32_t W) {
  if (n_tok < 1 || n_tok > kMaxTokens)
    return failf(SRS_ERR_INVALID, "n_tokens %lld outside 1..%lld", (long long)n_tok, (long long)kMaxTokens);
  if (W < 1 || W > kMaxWords) return failf(SRS_ERR_INVALID, "n_words %d outside 1..%d", W, kMaxWords);
  if (!tok || !hash) return failf(SRS_ERR_INVALID, "null tokens or hashes");
  std::vector<uint8_t> seen(W, 0);
  for (int64_t i = 0; i < n_tok; ++i) {
    if (tok[i] < 0 || tok[i] >= W)
      return failf(SRS_ERR_INVALID, "token %lld: word %d outside 0..%d", (long long)i, tok[i], W - 1);
    seen[tok[i]] = 1;
  }
  for (int w = 0; w < W; ++w)
    if (!seen[w]) return failf(SRS_ERR_INVALID, "word %d never occurs", w);
  std::vector<uint64_t> keys(W);
  for (int w = 0; w < W; ++w) keys[w] = trie_key(hash[w]);
  std::sort(keys.begin(), keys.end());
  for (int w = 1; w < W; ++w)
    if (keys[w] == keys[w - 1])
      return failf(SRS_ERR_INVALID, "two words share improve(hashCode); their hash-trie order is not supported");
  return SRS_OK;
}

// QuantileDiscretizer.fit's probabilities, `(0.0 to 1.0 by 1.0 / N).toArray`: a Scala 2.11 NumericRange[Double]
// (DoubleAsIfIntegral).  Its length is (BigDecimal(1.0) quot BigDecimal(step)) + 1, BigDecimal(d) being the decimal
// that Double.toString prints (taken here as the shortest decimal that reads back as d), and its element k is
// 0.0 + step * k.  When that decimal exceeds 1 / N the range stops one short of 1.0 (N = 11: ten steps), and its
// last element becomes the +inf split.  Empty on a decimal this cannot read.
std::vector<double> discretizer_probabilities(int num_buckets) {
  const double step = 1.0 / (double)num_buckets;
  char buf[64];
  const auto res = std::to_chars(buf, buf + sizeof(buf), step, std::chars_format::scientific);
  std::vector<double> probs;
  if (res.ec != std::errc()) return probs;
  const char* e = std::find(buf, res.ptr, 'e');
  __int128 mant = 0;
  int digits = 0;
  for (const char* c = buf; c < e; ++c)
    if (*c >= '0' && *c <= '9') { mant = mant * 10 + (*c - '0'); ++digits; }
  const int exp10 = atoi(e + 1);
  const int places = digits - 1 - exp10;            // step = mant / 10^places
  if (mant <= 0 || places < 0 || places > 36) return probs;
  __int128 p10 = 1;
  for (int k = 0; k < places; ++k) p10 *= 10;
  const long long count = (long long)(p10 / mant) + 1;
  for (long long k = 0; k < count; ++k) probs.push_back(0.0 + step * (double)k);
  return probs;
}

uint64_t stream_key(uint64_t seed, uint64_t stream) { return splitmix(seed, stream); }

// the rows of each part of d_part (device, n) into rows (host), part after part, in input order: one stable radix
// sort of (part, row) over the part's 8 bits
int gather_parts(HostCall& r, const int8_t* d_part, int n, int n_parts, int32_t* rows, int64_t* part_counts) {
  uint8_t *d_key, *d_key2;
  int32_t *d_iota, *d_rows;
  unsigned long long* d_cnt;
  CUDA_TRY(r.sc.alloc(&d_key, n));
  CUDA_TRY(r.sc.alloc(&d_key2, n));
  CUDA_TRY(r.sc.alloc(&d_iota, n));
  CUDA_TRY(r.sc.alloc(&d_rows, n));
  CUDA_TRY(r.sc.alloc(&d_cnt, n_parts));
  CUDA_TRY(cudaMemsetAsync(d_cnt, 0, sizeof(unsigned long long) * n_parts, r.s));
  fj_part_count_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_part, n, n_parts, d_key, d_iota, d_cnt);
  LAUNCHED();
  CUB_RUN(r, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_key, d_key2, d_iota, d_rows, n, 0, 8, r.s));
  std::vector<unsigned long long> cnt(n_parts);
  CUDA_TRY(cudaMemcpyAsync(cnt.data(), d_cnt, sizeof(unsigned long long) * n_parts, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  unsigned long long total = 0;
  for (int j = 0; j < n_parts; ++j) total += cnt[j];
  if (total) CUDA_TRY(cudaMemcpyAsync(rows, d_rows, sizeof(int32_t) * total, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  for (int j = 0; j < n_parts; ++j) part_counts[j] = (int64_t)cnt[j];
  return SRS_OK;
}

}  // namespace
}  // namespace srs

using namespace srs;

extern "C" int srs_approx_quantile_host(const double* values, int64_t n, const double* probabilities,
                                        int32_t n_probabilities, double relative_error, int32_t device, double* out) {
  PROPAGATE(check_values(values, n, "approx_quantile"));
  PROPAGATE(check_eps(relative_error));
  if (n_probabilities < 1 || n_probabilities > kMaxProbs || !probabilities || !out)
    return failf(SRS_ERR_INVALID, "need 1..%d probabilities and an output", kMaxProbs);
  for (int q = 0; q < n_probabilities; ++q)
    if (!(probabilities[q] >= 0.0 && probabilities[q] <= 1.0))
      return failf(SRS_ERR_INVALID, "probability %d (%g) outside [0, 1]", q, probabilities[q]);
  HostCall r;
  PROPAGATE(r.begin(device));
  double *d_v, *d_out;
  PROPAGATE(r.upload(&d_v, values, (size_t)n));
  CUDA_TRY(r.sc.alloc(&d_out, n_probabilities));
  PROPAGATE(quantiles_of_values(r, d_v, (int)n, probabilities, n_probabilities, relative_error, d_out));
  CUDA_TRY(cudaMemcpyAsync(out, d_out, sizeof(double) * n_probabilities, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  return SRS_OK;
}

extern "C" int srs_quantile_discretizer_host(const double* values, int64_t n, int32_t num_buckets,
                                             double relative_error, int32_t device, double* splits, int32_t* n_splits,
                                             int32_t* buckets) {
  PROPAGATE(check_values(values, n, "quantile_discretizer"));
  PROPAGATE(check_eps(relative_error));
  if (num_buckets < 2 || num_buckets > kMaxBuckets)
    return failf(SRS_ERR_INVALID, "num_buckets %d outside 2..%d", num_buckets, kMaxBuckets);
  if (!splits || !n_splits) return failf(SRS_ERR_INVALID, "null output");
  const std::vector<double> probs = discretizer_probabilities(num_buckets);
  const int nq = (int)probs.size();
  if (nq < 2 || nq > num_buckets + 1)
    return failf(SRS_ERR_INVALID, "num_buckets %d: %d probabilities from the step's decimal", num_buckets, nq);
  HostCall r;
  PROPAGATE(r.begin(device));
  double *d_v, *d_q, *d_splits;
  int *d_ns, *d_err;
  uint8_t* d_dup;
  int32_t* d_b;
  PROPAGATE(r.upload(&d_v, values, (size_t)n));
  CUDA_TRY(r.sc.alloc(&d_q, nq));
  CUDA_TRY(r.sc.alloc(&d_splits, nq));
  CUDA_TRY(r.sc.alloc(&d_ns, 1));
  CUDA_TRY(r.sc.alloc(&d_err, 1));
  CUDA_TRY(r.sc.alloc(&d_dup, nq));
  CUDA_TRY(r.sc.alloc(&d_b, buckets ? (size_t)n : 1));
  PROPAGATE(quantiles_of_values(r, d_v, (int)n, probs.data(), nq, relative_error, d_q));
  fj_splits_kernel<<<1, 1024, 0, r.s>>>(d_q, nq, d_splits, d_ns, d_err, d_dup);
  LAUNCHED();
  if (buckets) {
    fj_bucket_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_v, (int)n, d_splits, d_ns, d_b);
    LAUNCHED();
  }
  int ns = 0, err = 0;
  std::vector<double> h_splits(nq);
  CUDA_TRY(cudaMemcpyAsync(&ns, d_ns, sizeof(int), cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(&err, d_err, sizeof(int), cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(h_splits.data(), d_splits, sizeof(double) * nq, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  if (err)
    return failf(SRS_ERR_INVALID, "the %d distinct splits are not >= 3 strictly increasing values (Bucketizer)", ns);
  if (buckets) {
    CUDA_TRY(cudaMemcpyAsync(buckets, d_b, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, r.s));
    CUDA_TRY(cudaStreamSynchronize(r.s));
  }
  std::copy(h_splits.begin(), h_splits.begin() + ns, splits);
  *n_splits = ns;
  return SRS_OK;
}

extern "C" int srs_bucketize_host(const double* splits, int32_t n_splits, const double* values, int64_t n,
                                  int32_t device, int32_t* buckets) {
  PROPAGATE(check_splits(splits, n_splits));
  PROPAGATE(check_values(values, n, "bucketize"));
  if (!buckets) return failf(SRS_ERR_INVALID, "null output");
  const uint64_t lo = order_key(splits[0]), hi = order_key(splits[n_splits - 1]);
  for (int64_t i = 0; i < n; ++i) {
    const uint64_t k = order_key(values[i]);
    if (values[i] != splits[n_splits - 1] && (k < lo || k > hi))
      return failf(SRS_ERR_INVALID, "value %lld (%g) outside the splits [%g, %g]", (long long)i, values[i], splits[0],
                     splits[n_splits - 1]);
  }
  HostCall r;
  PROPAGATE(r.begin(device));
  double *d_v, *d_s;
  int* d_ns;
  int32_t* d_b;
  PROPAGATE(r.upload(&d_v, values, (size_t)n));
  PROPAGATE(r.upload(&d_s, splits, (size_t)n_splits));
  PROPAGATE(r.upload(&d_ns, &n_splits, 1));
  CUDA_TRY(r.sc.alloc(&d_b, n));
  fj_bucket_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_v, (int)n, d_s, d_ns, d_b);
  LAUNCHED();
  CUDA_TRY(cudaMemcpyAsync(buckets, d_b, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  return SRS_OK;
}

extern "C" int srs_minmax_scale_host(const double* values, int64_t n, const double* fit_min_max, int32_t device,
                                     double* out, double* min_max) {
  PROPAGATE(check_values(values, n, "minmax_scale"));
  if (!out) return failf(SRS_ERR_INVALID, "null output");
  if (fit_min_max && (std::isnan(fit_min_max[0]) || std::isnan(fit_min_max[1])))
    return failf(SRS_ERR_INVALID, "fitted min / max is NaN");
  HostCall r;
  PROPAGATE(r.begin(device));
  double *d_v, *d_out;
  uint64_t *d_keys, *d_kmm;
  PROPAGATE(r.upload(&d_v, values, (size_t)n));
  CUDA_TRY(r.sc.alloc(&d_out, n));
  CUDA_TRY(r.sc.alloc(&d_kmm, 2));
  if (fit_min_max) {
    const uint64_t k[2] = {order_key(fit_min_max[0]), order_key(fit_min_max[1])};
    CUDA_TRY(cudaMemcpyAsync(d_kmm, k, sizeof(k), cudaMemcpyHostToDevice, r.s));
    CUDA_TRY(cudaStreamSynchronize(r.s));         // k lives on this stack frame
  } else {
    CUDA_TRY(r.sc.alloc(&d_keys, n));
    fj_keys_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_v, (int)n, d_keys);
    LAUNCHED();
    CUB_RUN(r, cub::DeviceReduce::Min(tmp__, tb__, d_keys, d_kmm, (int)n, r.s));
    CUB_RUN(r, cub::DeviceReduce::Max(tmp__, tb__, d_keys, d_kmm + 1, (int)n, r.s));
  }
  fj_scale_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_v, (int)n, d_kmm, d_kmm + 1, d_out);
  LAUNCHED();
  uint64_t kmm[2];
  CUDA_TRY(cudaMemcpyAsync(kmm, d_kmm, sizeof(kmm), cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(out, d_out, sizeof(double) * n, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  if (min_max) {
    min_max[0] = key_value(kmm[0]);
    min_max[1] = key_value(kmm[1]);
  }
  return SRS_OK;
}

extern "C" int srs_rating_features_host(const int32_t* movie_id, const int8_t* half, int64_t n_ratings,
                                        int32_t device, int32_t capacity, int32_t* movie_ids, int64_t* counts,
                                        double* avg, double* var, int32_t* n_movies) {
  if (n_ratings < 1 || n_ratings > kMaxRatings)
    return failf(SRS_ERR_INVALID, "n_ratings %lld outside 1..%lld", (long long)n_ratings, (long long)kMaxRatings);
  if (!movie_id || !half) return failf(SRS_ERR_INVALID, "null ratings");
  if (!movie_ids || !counts || !avg || !var || !n_movies || capacity < 1)
    return failf(SRS_ERR_INVALID, "null output or capacity < 1");
  int32_t top = 0;
  for (int64_t i = 0; i < n_ratings; ++i) {
    if (movie_id[i] < 0 || movie_id[i] > kMaxMovieId)
      return failf(SRS_ERR_INVALID, "rating %lld: movie id %d outside 0..%d", (long long)i, movie_id[i], kMaxMovieId);
    if (half[i] < 1 || half[i] > 10)
      return failf(SRS_ERR_INVALID, "rating %lld: %d half-stars is not a rating in [0.5, 5]", (long long)i,
                     (int)half[i]);
    top = std::max(top, movie_id[i]);
  }
  const int n = (int)n_ratings, slots = top + 1;
  HostCall r;
  PROPAGATE(r.begin(device));
  int32_t *d_movie, *d_iota, *d_slot, *d_ids;
  int8_t* d_half;
  unsigned long long* d_mmom;
  uint8_t* d_flag;
  int* d_count;
  int64_t* d_cnt;
  double *d_avg, *d_var;
  PROPAGATE(r.upload(&d_movie, movie_id, n));
  PROPAGATE(r.upload(&d_half, half, n));
  CUDA_TRY(r.sc.alloc(&d_iota, n));
  CUDA_TRY(r.sc.alloc(&d_mmom, 3 * (size_t)slots));
  CUDA_TRY(r.sc.alloc(&d_slot, slots));
  CUDA_TRY(r.sc.alloc(&d_flag, slots));
  CUDA_TRY(r.sc.alloc(&d_ids, slots));
  CUDA_TRY(r.sc.alloc(&d_count, 1));
  CUDA_TRY(r.sc.alloc(&d_cnt, slots));
  CUDA_TRY(r.sc.alloc(&d_avg, slots));
  CUDA_TRY(r.sc.alloc(&d_var, slots));
  CUDA_TRY(cudaMemsetAsync(d_mmom, 0, sizeof(unsigned long long) * 3 * slots, r.s));
  CUDA_TRY(launch_movie_moments(d_movie, d_half, n, d_iota, d_mmom, r.s));
  fj_rated_kernel<<<grid_for(slots, 256), 256, 0, r.s>>>(d_mmom, slots, d_slot, d_flag);
  LAUNCHED();
  CUB_RUN(r, cub::DeviceSelect::Flagged(tmp__, tb__, d_slot, d_flag, d_ids, d_count, slots, r.s));
  fj_rating_kernel<<<grid_for(slots, 256), 256, 0, r.s>>>(d_mmom, d_ids, d_count, d_cnt, d_avg, d_var);
  LAUNCHED();
  int m = 0;
  CUDA_TRY(cudaMemcpyAsync(&m, d_count, sizeof(int), cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  if (m > capacity) return failf(SRS_ERR_RANGE, "%d rated movies exceed the capacity %d", m, capacity);
  CUDA_TRY(cudaMemcpyAsync(movie_ids, d_ids, sizeof(int32_t) * m, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(counts, d_cnt, sizeof(int64_t) * m, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(avg, d_avg, sizeof(double) * m, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(var, d_var, sizeof(double) * m, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  *n_movies = m;
  return SRS_OK;
}

extern "C" int srs_string_indexer_host(const int32_t* tokens, int64_t n_tokens, const int32_t* word_hash,
                                       int32_t n_words, int32_t device, int32_t* label_words, int64_t* label_counts) {
  PROPAGATE(check_tokens(tokens, n_tokens, word_hash, n_words));
  if (!label_words || !label_counts) return failf(SRS_ERR_INVALID, "null output");
  HostCall r;
  PROPAGATE(r.begin(device));
  int32_t *d_tok, *d_label_of, *d_label_word;
  int64_t* d_label_cnt;
  PROPAGATE(r.upload(&d_tok, tokens, (size_t)n_tokens));
  PROPAGATE(index_labels(r, d_tok, (int)n_tokens, word_hash, n_words, &d_label_of, &d_label_word, &d_label_cnt));
  CUDA_TRY(cudaMemcpyAsync(label_words, d_label_word, sizeof(int32_t) * n_words, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(label_counts, d_label_cnt, sizeof(int64_t) * n_words, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  return SRS_OK;
}

extern "C" int srs_genre_multihot_host(const int32_t* movie_id, const int32_t* offsets, const int32_t* words,
                                       int32_t n_movies, const int32_t* word_hash, int32_t n_words, int32_t device,
                                       int32_t* label_words, int64_t* label_counts, int32_t* out_movie_ids,
                                       int32_t* out_offsets, int32_t* out_indices) {
  if (n_movies < 1 || n_movies > kMaxMovieId + 1)
    return failf(SRS_ERR_INVALID, "n_movies %d outside 1..%d", n_movies, kMaxMovieId + 1);
  if (!movie_id || !offsets) return failf(SRS_ERR_INVALID, "null movies");
  if (!label_words || !label_counts || !out_movie_ids || !out_offsets || !out_indices)
    return failf(SRS_ERR_INVALID, "null output");
  if (offsets[0] != 0) return failf(SRS_ERR_INVALID, "offsets[0] must be 0");
  std::vector<uint8_t> id_seen((size_t)kMaxMovieId + 1, 0);
  for (int r = 0; r < n_movies; ++r) {
    const int len = offsets[r + 1] - offsets[r];
    if (len < 1 || len > kMaxWordsPerRow)
      return failf(SRS_ERR_INVALID, "movie row %d: %d words, need 1..%d", r, len, kMaxWordsPerRow);
    if (movie_id[r] < 0 || movie_id[r] > kMaxMovieId)
      return failf(SRS_ERR_INVALID, "movie row %d: id %d outside 0..%d", r, movie_id[r], kMaxMovieId);
    if (id_seen[movie_id[r]]++) return failf(SRS_ERR_INVALID, "movie %d listed twice", movie_id[r]);
  }
  const int64_t nnz = offsets[n_movies];
  PROPAGATE(check_tokens(words, nnz, word_hash, n_words));
  for (int r = 0; r < n_movies; ++r)
    for (int a = offsets[r]; a < offsets[r + 1]; ++a)
      for (int b = offsets[r]; b < a; ++b)
        if (words[a] == words[b]) return failf(SRS_ERR_INVALID, "movie %d lists a genre twice", movie_id[r]);
  HostCall r;
  PROPAGATE(r.begin(device));
  const int n = n_movies;
  int32_t *d_tok, *d_label_of, *d_label_word, *d_movie, *d_off, *d_iota, *d_order, *d_len, *d_ooff, *d_oidx;
  uint32_t *d_key, *d_key2;
  int64_t* d_label_cnt;
  PROPAGATE(r.upload(&d_tok, words, (size_t)nnz));
  PROPAGATE(r.upload(&d_movie, movie_id, n));
  PROPAGATE(r.upload(&d_off, offsets, (size_t)n + 1));
  CUDA_TRY(r.sc.alloc(&d_iota, n));
  CUDA_TRY(r.sc.alloc(&d_order, n));
  CUDA_TRY(r.sc.alloc(&d_key, n));
  CUDA_TRY(r.sc.alloc(&d_key2, n));
  CUDA_TRY(r.sc.alloc(&d_len, n));
  CUDA_TRY(r.sc.alloc(&d_ooff, (size_t)n + 1));
  CUDA_TRY(r.sc.alloc(&d_oidx, (size_t)nnz));
  PROPAGATE(index_labels(r, d_tok, (int)nnz, word_hash, n_words, &d_label_of, &d_label_word, &d_label_cnt));
  fj_row_iota_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_movie, n, d_key, d_iota);
  LAUNCHED();
  CUB_RUN(r, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_key, d_key2, d_iota, d_order, n, 0, 24, r.s));
  fj_row_len_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_order, d_off, n, d_len);
  LAUNCHED();
  CUDA_TRY(cudaMemsetAsync(d_ooff, 0, sizeof(int32_t), r.s));
  CUB_RUN(r, cub::DeviceScan::InclusiveSum(tmp__, tb__, d_len, d_ooff + 1, n, r.s));
  fj_csr_kernel<<<grid_for(n, 128), 128, 0, r.s>>>(d_order, d_off, d_tok, d_label_of, n, d_ooff, d_oidx);
  LAUNCHED();
  CUDA_TRY(cudaMemcpyAsync(label_words, d_label_word, sizeof(int32_t) * n_words, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(label_counts, d_label_cnt, sizeof(int64_t) * n_words, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(out_movie_ids, d_key2, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(out_offsets, d_ooff, sizeof(int32_t) * ((size_t)n + 1), cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaMemcpyAsync(out_indices, d_oidx, sizeof(int32_t) * nnz, cudaMemcpyDeviceToHost, r.s));
  CUDA_TRY(cudaStreamSynchronize(r.s));
  return SRS_OK;
}

extern "C" int srs_sample_split_host(int64_t n, uint64_t seed, double fraction, const double* weights,
                                     int32_t n_parts, int32_t device, int32_t* rows, int64_t* part_counts) {
  if (n < 1 || n > kMaxValues) return failf(SRS_ERR_INVALID, "n %lld outside 1..%lld", (long long)n,
                                              (long long)kMaxValues);
  if (!(fraction >= 0.0 && fraction <= 1.0)) return failf(SRS_ERR_INVALID, "fraction %g outside [0, 1]", fraction);
  if (n_parts < 1 || n_parts > kMaxParts || !weights)
    return failf(SRS_ERR_INVALID, "need 1..%d weights", kMaxParts);
  if (!rows || !part_counts) return failf(SRS_ERR_INVALID, "null output");
  double total = 0.0;
  for (int j = 0; j < n_parts; ++j) {
    if (!std::isfinite(weights[j]) || weights[j] < 0)
      return failf(SRS_ERR_INVALID, "weight %d (%g) is not finite and >= 0", j, weights[j]);
    total += weights[j];
  }
  if (!(total > 0.0)) return failf(SRS_ERR_INVALID, "the weights sum to 0");
  Bounds b{};
  for (int j = 0; j < n_parts; ++j) b.b[j + 1] = b.b[j] + weights[j] / total;
  HostCall r;
  PROPAGATE(r.begin(device));
  int8_t* d_part;
  CUDA_TRY(r.sc.alloc(&d_part, n));
  fj_part_kernel<<<grid_for(n, 256), 256, 0, r.s>>>((int)n, stream_key(seed, 0), stream_key(seed, 1), fraction, b,
                                                    n_parts, d_part);
  LAUNCHED();
  return gather_parts(r, d_part, (int)n, n_parts, rows, part_counts);
}

extern "C" int srs_sample_split_by_timestamp_host(const int64_t* timestamp, int64_t n, uint64_t seed, double fraction,
                                                  double relative_error, int32_t device, int32_t* rows,
                                                  int64_t* part_counts, double* split_timestamp) {
  if (n < 1 || n > kMaxValues) return failf(SRS_ERR_INVALID, "n %lld outside 1..%lld", (long long)n,
                                              (long long)kMaxValues);
  if (!timestamp) return failf(SRS_ERR_INVALID, "null timestamps");
  if (!(fraction >= 0.0 && fraction <= 1.0)) return failf(SRS_ERR_INVALID, "fraction %g outside [0, 1]", fraction);
  PROPAGATE(check_eps(relative_error));
  if (!rows || !part_counts || !split_timestamp) return failf(SRS_ERR_INVALID, "null output");
  for (int64_t i = 0; i < n; ++i)
    if (timestamp[i] < -(1ll << 53) || timestamp[i] > (1ll << 53))
      return failf(SRS_ERR_INVALID, "timestamp %lld outside -2^53..2^53, where a double is exact",
                   (long long)timestamp[i]);
  HostCall r;
  PROPAGATE(r.begin(device));
  const int nn = (int)n;
  int64_t* d_ts;
  uint64_t* d_keys;
  uint8_t* d_flag;
  int* d_count;
  int8_t* d_part;
  double *d_prob, *d_split;
  const double p08 = 0.8;
  PROPAGATE(r.upload(&d_ts, timestamp, (size_t)n));
  CUDA_TRY(r.sc.alloc(&d_keys, n));
  CUDA_TRY(r.sc.alloc(&d_flag, n));
  CUDA_TRY(r.sc.alloc(&d_count, 1));
  CUDA_TRY(r.sc.alloc(&d_part, n));
  PROPAGATE(r.upload(&d_prob, &p08, 1));
  CUDA_TRY(r.sc.alloc(&d_split, 1));
  CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int), r.s));
  fj_ts_keys_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_ts, nn, stream_key(seed, 0), fraction, d_keys, d_flag);
  LAUNCHED();
  fj_flag_count_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_flag, nn, d_count);
  LAUNCHED();
  PROPAGATE(quantiles_of_keys(r, d_keys, nn, d_count, d_prob, 1, relative_error, d_split));
  fj_ts_part_kernel<<<grid_for(n, 256), 256, 0, r.s>>>(d_ts, d_flag, nn, d_split, d_part);
  LAUNCHED();
  double split = 0.0;
  CUDA_TRY(cudaMemcpyAsync(&split, d_split, sizeof(double), cudaMemcpyDeviceToHost, r.s));
  PROPAGATE(gather_parts(r, d_part, nn, 2, rows, part_counts));
  *split_timestamp = split;
  return SRS_OK;
}
