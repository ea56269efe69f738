// featureeng.cu - the reference's sample builder (FeatureEngForRecModel.scala:21-130) on one device.
//
// ratings (userId, movieId, half-star rating, timestamp) + a per-movie table (release year from the title, genre
// word indices in string order) -> the 27-column sample rows every model here reads, in ratings file order, rows
// with fewer than two earlier ratings of the same user dropped.  DESIGN.md section 4.11 gives the semantics.
//
// Launches, all on one stream, with no host round trip between them:
//   1. fe_prepare_kernel   the movies' exact integer moments (count, sum h, sum h^2 of half-stars; 64-bit
//                          integer atomics, so order-free);
//   2. user_time_order     sort keys (timestamp in *string* order), then two stable CUB radix sorts: by
//                          timestamp key, then by user - ties keep file order (item2vec.cu's sentences use it too);
//   3. fe_movie_kernel     per movie: count, format_number(avg), format_number(stddev);
//   4. fe_window_kernel    one thread per rating scans its <= 100 predecessors of the same user, oldest first;
//   5. CUB DeviceSelect    the kept rows (userRatingCount > 1), in file order;
//   6. fe_pack_kernel      every derived column of the kept rows.
// Averages and the movies' standard deviations come from exact integer moments (ratings are half-stars, years are
// integers): one correctly rounded double division of two integers below 2^53, then a correctly rounded sqrt.  A
// user window's standard deviations follow Spark's own value-by-value update in window order (Welford).
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"

namespace srs {
namespace {

constexpr int kWindow = 100;           // rowsBetween(-100, -1)
constexpr int kMaxGenres = 24;         // the UDF's HashMap is rehashed once (16 -> 32 buckets) at the 13th key
constexpr int kTsBits = 38;            // (timestamp left-aligned to 10 digits) << 4 | digits  <  10^10 * 16
constexpr int64_t kMaxRatings = 21000000;    // every movie's 20.25 n^2 bound on n S2 - S1^2 stays below 2^53
constexpr int32_t kMaxMovieSlots = 1 << 24;

struct GenreBuckets {                  // per genre word: its bucket in the UDF's 16- and 32-slot hash tables
  uint8_t b16[kMaxGenres], b32[kMaxGenres];
};

// java.text.DecimalFormat("#,##0.00") with HALF_EVEN on the exact binary value of x (>= 0): the k it prints as
// k/100.  100 x = p + e exactly (e from the fma), so the comparisons with the half-way point are exact.
__device__ __forceinline__ long long hundredths_half_even(double x) {
  const double p = __dmul_rn(100.0, x);
  const double e = fma(100.0, x, -p);
  const double k0 = floor(p);
  const double d = (p - k0) - 0.5;
  long long k = (long long)k0;
  if (d > -e || (d == -e && (k & 1))) ++k;
  return k;
}

// the float32 of the two-decimal text: the correctly rounded k / 100
__device__ __forceinline__ float format2(double x) {
  return __fdiv_rn((float)hundredths_half_even(x), 100.f);
}

// sqrt(Q / (4 n (n - 1))), Q = n S2 - S1^2 in half-stars; 0 for n < 2 (stddev_samp's NaN / null, then na.fill(0))
__device__ __forceinline__ double stddev_exact(long long n, long long s1, long long s2) {
  if (n < 2) return 0.0;
  const long long q = n * s2 - s1 * s1;
  return sqrt(__ddiv_rn((double)q, (double)(4 * n * (n - 1))));
}

// stddev_samp as Spark's CentralMomentAgg updates it, value by value, one rounding per operation (no fused
// multiply-add): a user window has a defined order, and this rounding decides some HALF_EVEN ties of the output.
struct Welford {
  double n = 0.0, avg = 0.0, m2 = 0.0;
  __device__ __forceinline__ void add(double x) {
    const double nn = __dadd_rn(n, 1.0);
    const double delta = __dsub_rn(x, avg);
    const double delta_n = __ddiv_rn(delta, nn);
    avg = __dadd_rn(avg, delta_n);
    m2 = __dadd_rn(m2, __dmul_rn(delta, __dsub_rn(delta, delta_n)));
    n = nn;
  }
  __device__ __forceinline__ double stddev() const {      // n < 2: NaN / null, then na.fill(0)
    return n >= 2.0 ? sqrt(__ddiv_rn(m2, __dsub_rn(n, 1.0))) : 0.0;
  }
};

__global__ void fe_ts_key_kernel(const int32_t* __restrict__ ts, int n, uint64_t* __restrict__ ts_key,
                                 int32_t* __restrict__ iota) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int64_t t = ts[i];
    int digits = 1;
    int64_t p10 = 10;
    while (p10 <= t) { p10 *= 10; ++digits; }
    int64_t aligned = t;
    for (int d = digits; d < 10; ++d) aligned *= 10;
    ts_key[i] = ((uint64_t)aligned << 4) | (uint64_t)digits;   // a string prefix sorts first
    iota[i] = i;
  }
}

__global__ void fe_prepare_kernel(const int32_t* __restrict__ movie, const int8_t* __restrict__ half, int n,
                                  int32_t* __restrict__ iota, unsigned long long* __restrict__ mmom) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    iota[i] = i;
    const unsigned long long h = (unsigned long long)half[i];
    unsigned long long* m = mmom + 3 * (size_t)movie[i];
    atomicAdd(m, 1ull);
    atomicAdd(m + 1, h);
    atomicAdd(m + 2, h * h);
  }
}

__global__ void fe_gather_user_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ user, int n,
                                      uint32_t* __restrict__ ukey) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    ukey[i] = (uint32_t)user[order[i]];
}

__global__ void fe_movie_kernel(const unsigned long long* __restrict__ mmom, int slots, int32_t* __restrict__ mcount,
                                float* __restrict__ mavg, float* __restrict__ mstd) {
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < slots; m += gridDim.x * blockDim.x) {
    const long long c = (long long)mmom[3 * (size_t)m], s1 = (long long)mmom[3 * (size_t)m + 1],
                    s2 = (long long)mmom[3 * (size_t)m + 2];
    mcount[m] = (int32_t)c;
    mavg[m] = c ? format2(__ddiv_rn((double)s1 * 0.5, (double)c)) : 0.f;
    mstd[m] = format2(stddev_exact(c, s1, s2));
  }
}

// One thread per rating in (user, timestamp string, file index) order; results go to file position order[i].
__global__ void fe_window_kernel(const int32_t* __restrict__ order, const uint32_t* __restrict__ suser,
                                 const int32_t* __restrict__ movie, const int8_t* __restrict__ half, int n,
                                 const int32_t* __restrict__ movie_year, const int32_t* __restrict__ movie_genres,
                                 int L, int G, GenreBuckets gb, int32_t* __restrict__ w_count,
                                 float* __restrict__ w_f32 /* [4][n] */, int32_t* __restrict__ w_rated /* [n][5] */,
                                 int32_t* __restrict__ w_genre /* [n][5] */, uint8_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t u = suser[i];
  int lo = i;
  while (lo > 0 && i - lo < kWindow && suser[lo - 1] == u) --lo;
  uint16_t cnt[kMaxGenres];
  uint8_t ins[kMaxGenres];
  for (int g = 0; g < G; ++g) cnt[g] = 0;
  int nd = 0;
  long long s1 = 0, y1 = 0;
  Welford wr, wy;
  int rated[5] = {0, 0, 0, 0, 0};
  for (int j = lo; j < i; ++j) {                       // oldest first: collect_list's order
    const int f = __ldg(order + j);
    const int m = __ldg(movie + f);
    const long long h = __ldg(half + f), y = __ldg(movie_year + m);
    s1 += h; y1 += y;
    wr.add(__dmul_rn((double)h, 0.5));
    wy.add((double)y);
    if (h >= 7) {                                      // label: rating >= 3.5
      rated[4] = rated[3]; rated[3] = rated[2]; rated[2] = rated[1]; rated[1] = rated[0]; rated[0] = m;
      for (int p = 0; p < L; ++p) {
        const int g = __ldg(movie_genres + (size_t)m * L + p);
        if (g < 0) break;
        if (cnt[g]++ == 0) ins[g] = (uint8_t)nd++;   // the HashMap's insertion order
      }
    }
  }
  const long long c = i - lo;
  const int fi = __ldg(order + i);
  w_count[fi] = (int32_t)c;
  keep[fi] = c > 1;
  w_f32[fi] = c ? (float)(int)__ddiv_rn((double)y1, (double)c) : 0.f;          // avg(...).cast(IntegerType)
  w_f32[(size_t)n + fi] = format2(wy.stddev());
  w_f32[2 * (size_t)n + fi] = c ? format2(__ddiv_rn((double)s1 * 0.5, (double)c)) : 0.f;
  w_f32[3 * (size_t)n + fi] = format2(wr.stddev());
#pragma unroll
  for (int k = 0; k < 5; ++k) w_rated[(size_t)fi * 5 + k] = rated[k];
  // sortWith(count desc) is stable over the HashMap's iteration order: buckets high to low, each bucket head first
  // (newest first); past 12 keys the table was rehashed at the 13th, which reversed the older keys' order.
  uint32_t taken = 0;
  for (int k = 0; k < 5; ++k) {
    int best = -1;
    uint64_t bkey = ~0ull;
    for (int g = 0; g < G; ++g) {
      if (!cnt[g] || (taken >> g & 1)) continue;
      const uint32_t r = ins[g];
      const uint32_t it = nd <= 12 ? ((15u - gb.b16[g]) << 8) | (255u - r)
                                   : ((31u - gb.b32[g]) << 16) |
                                         (r >= 13 ? 255u - r : (1u << 15) | ((uint32_t)gb.b16[g] << 8) | r);
      const uint64_t key = ((uint64_t)(65535u - cnt[g]) << 32) | it;
      if (key < bkey) { bkey = key; best = g; }
    }
    if (best >= 0) taken |= 1u << best;
    w_genre[(size_t)fi * 5 + k] = best;
  }
}

__global__ void fe_pack_kernel(const int32_t* __restrict__ kept, const int* __restrict__ n_kept, int n,
                               const int32_t* __restrict__ movie, const int8_t* __restrict__ half,
                               const int32_t* __restrict__ movie_year, const int32_t* __restrict__ movie_genres, int L,
                               const int32_t* __restrict__ mcount, const float* __restrict__ mavg,
                               const float* __restrict__ mstd, const int32_t* __restrict__ w_count,
                               const float* __restrict__ w_f32, const int32_t* __restrict__ w_rated,
                               const int32_t* __restrict__ w_genre, int32_t* __restrict__ o_i32 /* [5][n] */,
                               int32_t* __restrict__ o_mgenre /* [n][3] */,
                               float* __restrict__ o_f32 /* [6][n] */, int32_t* __restrict__ o_rated,
                               int32_t* __restrict__ o_genre) {
  const int total = *n_kept;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
    const int f = kept[k], m = movie[f];
    o_i32[k] = f;
    o_i32[(size_t)n + k] = half[f] >= 7;
    o_i32[2 * (size_t)n + k] = movie_year[m];
    o_i32[3 * (size_t)n + k] = mcount[m];
    o_i32[4 * (size_t)n + k] = w_count[f];
    for (int p = 0; p < 3; ++p) o_mgenre[(size_t)k * 3 + p] = p < L ? movie_genres[(size_t)m * L + p] : -1;
    o_f32[k] = mavg[m];
    o_f32[(size_t)n + k] = mstd[m];
    for (int c = 0; c < 4; ++c) o_f32[(2 + c) * (size_t)n + k] = w_f32[c * (size_t)n + f];
    for (int c = 0; c < 5; ++c) {
      o_rated[(size_t)k * 5 + c] = w_rated[(size_t)f * 5 + c];
      o_genre[(size_t)k * 5 + c] = w_genre[(size_t)f * 5 + c];
    }
  }
}

// scala.collection.mutable.HashTable.index for a String key: byteswap32(hashCode), rotated right by the seed
// bitCount(15) = 4 fixed at construction, then the top log2(len) bits.
uint8_t hash_bucket(int32_t hash_code, int log2_len) {
  uint32_t hc = (uint32_t)hash_code * 0x9E3775CDu;
  hc = __builtin_bswap32(hc);
  hc *= 0x9E3775CDu;
  const uint32_t rot = (hc >> 4) | (hc << 28);
  return (uint8_t)(rot >> (32 - log2_len));
}

// user_time_order's temporaries: stream-ordered allocations, handed back to the device's pool when the function
// returns, so they are not held until the call ends.  With cudaMalloc / cudaFree instead, build_samples over 20 M
// ratings measured 6.80 s against 6.27 s (medians of 4 calls, H100 80GB HBM3 at a 700 W power limit).
struct PoolTemps {
  cudaStream_t s;
  std::vector<void*> ptrs;
  ~PoolTemps() { for (void* p : ptrs) cudaFreeAsync(p, s); }
  template <class T>
  cudaError_t alloc(T** p, size_t count) {
    void* q = nullptr;
    const cudaError_t e = cudaMallocAsync(&q, (count ? count : 1) * sizeof(T), s);
    if (e == cudaSuccess) ptrs.push_back(q);
    *p = static_cast<T*>(q);
    return e;
  }
};

}  // namespace

int user_time_order(cudaStream_t s, const int32_t* d_user, const int32_t* d_ts, int n, int32_t* d_order,
                    uint32_t* d_user_sorted) {
  if (n <= 0) return SRS_OK;
  PoolTemps t{s};
  uint64_t *tskey = nullptr, *tskey2 = nullptr;
  int32_t *iota = nullptr, *order = nullptr;
  uint32_t* ukey = nullptr;
  uint8_t* tmp;
  size_t tmp_ts = 0, tmp_u = 0;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_ts, tskey, tskey2, iota, order, n, 0, kTsBits, s));
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_u, ukey, d_user_sorted, order, d_order, n, 0, 31, s));
  CUDA_TRY(t.alloc(&tskey, n)); CUDA_TRY(t.alloc(&tskey2, n)); CUDA_TRY(t.alloc(&iota, n));
  CUDA_TRY(t.alloc(&order, n)); CUDA_TRY(t.alloc(&ukey, n)); CUDA_TRY(t.alloc(&tmp, std::max(tmp_ts, tmp_u)));
  const int T = 256;
  fe_ts_key_kernel<<<grid_for(n, T), T, 0, s>>>(d_ts, n, tskey, iota);
  LAUNCHED();
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_ts, tskey, tskey2, iota, order, n, 0, kTsBits, s));
  fe_gather_user_kernel<<<grid_for(n, T), T, 0, s>>>(order, d_user, n, ukey);
  LAUNCHED();
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_u, ukey, d_user_sorted, order, d_order, n, 0, 31, s));
  return SRS_OK;
}

cudaError_t launch_movie_moments(const int32_t* d_movie, const int8_t* d_half, int n, int32_t* d_iota,
                                 unsigned long long* d_mmom, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  const int T = 256;
  fe_prepare_kernel<<<grid_for(n, T), T, 0, s>>>(d_movie, d_half, n, d_iota, d_mmom);
  ++g_launch_count;
  return cudaGetLastError();
}

}  // namespace srs

using namespace srs;

extern "C" int srs_featureeng_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                                   const int32_t* timestamp, int64_t n_ratings, const int32_t* movie_year,
                                   const int32_t* movie_genres, int32_t n_movie_slots, int32_t genres_per_movie,
                                   const int32_t* genre_hash, int32_t n_genres, int32_t device, srs_samples* out,
                                   int64_t* n_kept) {
  if (!out || !n_kept) return failf(SRS_ERR_INVALID, "null output");
  *n_kept = 0;
  if (n_ratings < 0 || n_ratings > kMaxRatings)
    return failf(SRS_ERR_INVALID, "n_ratings %lld outside 0..%lld", (long long)n_ratings, (long long)kMaxRatings);
  if (n_movie_slots < 1 || n_movie_slots > kMaxMovieSlots)
    return failf(SRS_ERR_INVALID, "n_movie_slots %d outside 1..%d", n_movie_slots, kMaxMovieSlots);
  if (genres_per_movie < 1 || genres_per_movie > kMaxGenres || n_genres < 0 || n_genres > kMaxGenres)
    return failf(SRS_ERR_INVALID, "genres_per_movie must be in 1..%d and n_genres in 0..%d", kMaxGenres, kMaxGenres);
  if (n_ratings && (!user_id || !movie_id || !half || !timestamp)) return failf(SRS_ERR_INVALID, "null ratings");
  if (!movie_year || !movie_genres || (n_genres && !genre_hash)) return failf(SRS_ERR_INVALID, "null movie table");
  const int32_t* outs_i[] = {out->row, out->label, out->release_year, out->movie_genre, out->movie_rating_count,
                             out->user_rated_movie, out->user_rating_count, out->user_genre};
  const float* outs_f[] = {out->movie_avg_rating, out->movie_rating_stddev, out->user_avg_release_year,
                           out->user_release_year_stddev, out->user_avg_rating, out->user_rating_stddev};
  for (const int32_t* p : outs_i) if (!p) return failf(SRS_ERR_INVALID, "null output column");
  for (const float* p : outs_f) if (!p) return failf(SRS_ERR_INVALID, "null output column");
  const int n = (int)n_ratings;
  for (int i = 0; i < n; ++i) {
    if (user_id[i] < 0 || movie_id[i] < 0)
      return failf(SRS_ERR_INVALID, "rating %d: negative id (user %d, movie %d)", i, user_id[i], movie_id[i]);
    if (movie_id[i] >= n_movie_slots)
      return failf(SRS_ERR_INVALID, "rating %d: movie %d outside the movie table (%d slots)", i, movie_id[i],
                     n_movie_slots);
    if (half[i] < 1 || half[i] > 10)
      return failf(SRS_ERR_INVALID, "rating %d: %d half-stars is not a rating in [0.5, 5]", i, (int)half[i]);
    if (timestamp[i] <= 0) return failf(SRS_ERR_INVALID, "rating %d: timestamp %d is not positive", i, timestamp[i]);
  }
  const int L = genres_per_movie;
  for (int64_t m = 0; m < n_movie_slots; ++m) {
    if (movie_year[m] < -999 || movie_year[m] > 9999)
      return failf(SRS_ERR_INVALID, "movie %lld: release year %d is not four characters", (long long)m, movie_year[m]);
    bool ended = false;
    for (int p = 0; p < L; ++p) {
      const int g = movie_genres[m * L + p];
      if (g < -1 || g >= n_genres || (ended && g != -1))
        return failf(SRS_ERR_INVALID, "movie %lld: genre list must be word indices in 0..%d, then -1 padding",
                       (long long)m, n_genres - 1);
      ended |= g < 0;
    }
  }
  GenreBuckets gb{};
  for (int g = 0; g < n_genres; ++g) {
    gb.b16[g] = hash_bucket(genre_hash[g], 4);
    gb.b32[g] = hash_bucket(genre_hash[g], 5);
  }
  if (n == 0) return SRS_OK;

  HostCall c;
  PROPAGATE(c.begin(device));
  Scratch& sc = c.sc;
  cudaStream_t s = c.s;
  const size_t slots = (size_t)n_movie_slots;
  int32_t *d_user, *d_movie, *d_ts, *d_year, *d_genres, *d_iota, *d_order2, *d_mcount, *d_wcount;
  int32_t *d_wrated, *d_wgenre, *d_kept, *d_oi32, *d_omgenre, *d_orated, *d_ogenre;
  int8_t* d_half;
  uint32_t* d_ukey2;
  unsigned long long* d_mmom;
  float *d_mavg, *d_mstd, *d_wf32, *d_of32;
  uint8_t* d_keep;
  int* d_nkept;
  CUDA_TRY(sc.alloc(&d_user, n)); CUDA_TRY(sc.alloc(&d_movie, n)); CUDA_TRY(sc.alloc(&d_ts, n));
  CUDA_TRY(sc.alloc(&d_half, n)); CUDA_TRY(sc.alloc(&d_year, slots)); CUDA_TRY(sc.alloc(&d_genres, slots * L));
  CUDA_TRY(sc.alloc(&d_iota, n)); CUDA_TRY(sc.alloc(&d_order2, n)); CUDA_TRY(sc.alloc(&d_ukey2, n)); CUDA_TRY(sc.alloc(&d_mmom, 3 * slots)); CUDA_TRY(sc.alloc(&d_mcount, slots));
  CUDA_TRY(sc.alloc(&d_mavg, slots)); CUDA_TRY(sc.alloc(&d_mstd, slots)); CUDA_TRY(sc.alloc(&d_wcount, n));
  CUDA_TRY(sc.alloc(&d_wf32, 4 * (size_t)n)); CUDA_TRY(sc.alloc(&d_wrated, 5 * (size_t)n));
  CUDA_TRY(sc.alloc(&d_wgenre, 5 * (size_t)n)); CUDA_TRY(sc.alloc(&d_keep, n)); CUDA_TRY(sc.alloc(&d_kept, n));
  CUDA_TRY(sc.alloc(&d_nkept, 1)); CUDA_TRY(sc.alloc(&d_oi32, 5 * (size_t)n)); CUDA_TRY(sc.alloc(&d_omgenre, 3 * (size_t)n)); CUDA_TRY(sc.alloc(&d_of32, 6 * (size_t)n));
  CUDA_TRY(sc.alloc(&d_orated, 5 * (size_t)n)); CUDA_TRY(sc.alloc(&d_ogenre, 5 * (size_t)n));

  CUDA_TRY(cudaMemcpyAsync(d_user, user_id, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_movie, movie_id, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_ts, timestamp, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_half, half, n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_year, movie_year, sizeof(int32_t) * slots, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_genres, movie_genres, sizeof(int32_t) * slots * L, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemsetAsync(d_mmom, 0, sizeof(unsigned long long) * 3 * slots, s));

  const int T = 256;
  CUDA_TRY(launch_movie_moments(d_movie, d_half, n, d_iota, d_mmom, s));
  PROPAGATE(user_time_order(s, d_user, d_ts, n, d_order2, d_ukey2));
  fe_movie_kernel<<<grid_for(n_movie_slots, T), T, 0, s>>>(d_mmom, n_movie_slots, d_mcount, d_mavg, d_mstd);
  LAUNCHED();
  fe_window_kernel<<<(n + 127) / 128, 128, 0, s>>>(d_order2, d_ukey2, d_movie, d_half, n, d_year, d_genres, L,
                                                   n_genres, gb, d_wcount, d_wf32, d_wrated, d_wgenre, d_keep);
  LAUNCHED();
  CUB_RUN(c, cub::DeviceSelect::Flagged(tmp__, tb__, d_iota, d_keep, d_kept, d_nkept, n, s));
  fe_pack_kernel<<<grid_for(n, T), T, 0, s>>>(d_kept, d_nkept, n, d_movie, d_half, d_year, d_genres, L, d_mcount,
                                              d_mavg, d_mstd, d_wcount, d_wf32, d_wrated, d_wgenre, d_oi32, d_omgenre, d_of32,
                                              d_orated, d_ogenre);
  LAUNCHED();
  int kept = 0;
  CUDA_TRY(cudaMemcpyAsync(&kept, d_nkept, sizeof(int), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  int32_t* dst_i[] = {out->row, out->label, out->release_year, out->movie_rating_count, out->user_rating_count};
  for (int c = 0; c < 5; ++c)
    CUDA_TRY(cudaMemcpyAsync(dst_i[c], d_oi32 + (size_t)c * n, sizeof(int32_t) * kept, cudaMemcpyDeviceToHost, s));
  float* dst_f[] = {out->movie_avg_rating, out->movie_rating_stddev, out->user_avg_release_year,
                    out->user_release_year_stddev, out->user_avg_rating, out->user_rating_stddev};
  for (int c = 0; c < 6; ++c)
    CUDA_TRY(cudaMemcpyAsync(dst_f[c], d_of32 + (size_t)c * n, sizeof(float) * kept, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out->movie_genre, d_omgenre, sizeof(int32_t) * 3 * kept, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out->user_rated_movie, d_orated, sizeof(int32_t) * 5 * kept, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out->user_genre, d_ogenre, sizeof(int32_t) * 5 * kept, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  *n_kept = kept;
  return SRS_OK;
}
