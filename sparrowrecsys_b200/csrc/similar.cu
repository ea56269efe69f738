// similar.cu - the reference's "similar movies" page, SimilarMovieProcess.getRecList(movieId, size, model)
// (online/recprocess/SimilarMovieProcess.java:20-32), for many query movies per call, with either of its two
// candidate sources, and its embedding recall retrievalCandidatesByEmbedding (:91-112).  DESIGN.md sections 4.23
// and 4.24 give the semantics; oracle/similar_movies.py and oracle/similar_recall.py restate the Java.
//
// Catalogue (srs_similar_catalog_create_ex_host, once):
//   ratings   each rating's load-order slot (binary search of the sorted ids), a stable radix sort of (slot,
//             score), and sim_average_kernel: one thread per movie walks its ratings in file order with
//             Movie.addRating's running mean (avg * n + score) / (n + 1) in double, each operation rounded once;
//   by rating a stable radix sort of the movies by desc_key(average) (double_key.cuh): Double.compare descending,
//             ties in load order - the order getMoviesByGenre's stable List.sort gives every genre's sub-list;
//   genres    sim_genre_top_kernel: one block per genre keeps the first kGenreTop movies of that order that carry
//             the genre (a block scan per chunk), and sim_listed_kernel marks each movie with the genres whose
//             lists (and whose first kMultiGenreTop entries) hold it;
//   getMovies DataManager.movieMap's HashMap iteration order (the table length simulated on the host, a stable
//             radix sort of the slots by bucket), then stable radix sorts of that order by desc_key(average) and
//             by release year descending: the top kGlobalTop of each, the first kPool by rating, in id order, and
//             the first kRecForYou by rating in that order (recforyou.cu's candidates).
// Query (srs_similar_movies_candidates_host): sim_query_kernel, one block per query movie -
//   candidates the entries of the query's genre lists (GENRE), or their first kMultiGenreTop entries and the two
//             global top lists (MULTIPLE); an entry is kept unless it is the query or an earlier list of the
//             query holds it too, so each candidate appears once;
//   scores    calculateSimilarScore in double, or the emb ranker's cosine (cosine.cuh, shared with util.cu);
//   order     a bitonic sort in shared memory by (desc_key(score), movie id): score descending, ties by id.
// Embedding recall (srs_similar_embedding_recall_host): sim_emb_recall_kernel, one block per query movie, scores the
//   whole pool with the same cosine and block-radix-sorts it by ~desc_key(score): Double.compare ascending, ties
//   by movie id through the sort's stability over the id-ordered pool.
// No float atomics and every sum in a fixed order: the same inputs give the same bits.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <cstring>
#include <memory>
#include <new>
#include <vector>

#include "../../include/srs_ctr.h"
#include "cosine.cuh"
#include "double_key.cuh"
#include "hostcall.h"

struct srs_similar_catalog {
  int32_t device = 0;
  int32_t n_movies = 0, n_genres = 0, dim = 0;
  int32_t max_cands = 0;                 // the largest candidate list (before the query is removed) of any movie
  int32_t* ids_sorted = nullptr;         // [n_movies] ascending movie id ...
  int32_t* slot_sorted = nullptr;        // ... and its load-order slot
  int32_t* movie_id = nullptr;           // [n_movies] by slot
  uint64_t* mask = nullptr;              // [n_movies] the movie's genres
  uint64_t* listed = nullptr;            // [n_movies] the genres whose top lists hold the movie
  double* avg = nullptr;                 // [n_movies] Movie.averageRating
  int32_t* glist = nullptr;              // [n_genres][kGenreTop] slots, best first
  int32_t* gcnt = nullptr;               // [n_genres]
  float* emb = nullptr;                  // [n_emb][dim]
  int32_t* emb_row = nullptr;            // [n_movies] the movie's row of emb, -1 for none
  // getMovies(size, sortBy) (DataManager.java:271-283): movieMap's iteration order, known unless a bin is treeified
  bool hash_order = false;
  bool has_year = false;                 // created with release years: multi-channel recall is possible
  int32_t max_multi = 0;                 // the largest multi-channel candidate list (before the query is removed)
  int32_t n_top = 0, n_pool = 0;         // entries of rtop / ytop (0 without years), of pool
  uint64_t* listed_multi = nullptr;      // [n_movies] the genres whose first kMultiGenreTop entries hold the movie
  uint8_t* in_rtop = nullptr;            // [n_movies] 1 when getMovies(100, "rating") holds the movie
  int32_t* rtop = nullptr;               // [n_top] getMovies(100, "rating"), slots
  int32_t* ytop = nullptr;               // [n_top] getMovies(100, "releaseYear"), slots
  int32_t* pool = nullptr;               // [n_pool] getMovies(10000, "rating"), slots in ascending movie id
  int32_t n_rec = 0;                     // entries of rec
  int32_t* rec = nullptr;                // [n_rec] getMovies(800, "rating"), slots in that order (RecForYouProcess)
  ~srs_similar_catalog() {
    cudaSetDevice(device);
    for (void* p : {(void*)ids_sorted, (void*)slot_sorted, (void*)movie_id, (void*)mask, (void*)listed, (void*)avg,
                    (void*)glist, (void*)gcnt, (void*)emb, (void*)emb_row, (void*)listed_multi, (void*)in_rtop,
                    (void*)rtop, (void*)ytop, (void*)pool, (void*)rec})
      cudaFree(p);
  }
};

namespace srs {
namespace {

constexpr int kGenreTop = 100;           // getMoviesByGenre(genre, 100, "rating"): SimilarMovieProcess.java:42
constexpr int kMaxGenres = 64;           // one bit each in a uint64 mask
constexpr int kMultiGenreTop = 20;       // getMoviesByGenre(genre, 20, "rating"): SimilarMovieProcess.java:65
constexpr int kGlobalTop = 100;          // getMovies(100, "rating" / "releaseYear"): :71, :76
constexpr int kPool = 10000;             // getMovies(10000, "rating"): :96
constexpr int kRecForYou = 800;          // getMovies(800, "rating"): RecForYouProcess.java:34-35
constexpr int kThreads = 256;
constexpr int kQueryThreads = 256;
constexpr int kSegRating = -1, kSegYear = -2;   // sim_query_kernel's segments of the two global lists

#define SIM_GRID_STRIDE(i, n) \
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// load-order slot of movie `id`, -1 when the catalogue does not hold it
__device__ __forceinline__ int find_slot(const int32_t* __restrict__ ids, const int32_t* __restrict__ slots, int n,
                                         int32_t id) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ids[mid] < id) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && ids[lo] == id ? slots[lo] : -1;
}

__global__ void sim_iota_kernel(int32_t* __restrict__ x, int n) {
  SIM_GRID_STRIDE(i, n) x[i] = (int32_t)i;
}

// each rating's movie slot; ratings of movies outside the catalogue get n_movies and sort last
__global__ void sim_rating_slot_kernel(const int32_t* __restrict__ movie, int64_t n, const int32_t* __restrict__ ids,
                                       const int32_t* __restrict__ slots, int n_movies, int32_t* __restrict__ out) {
  SIM_GRID_STRIDE(i, n) {
    const int s = find_slot(ids, slots, n_movies, movie[i]);
    out[i] = s < 0 ? n_movies : s;
  }
}

// first index of `slot` in the ascending rslot[0 .. n)
__device__ __forceinline__ int64_t lower_bound(const int32_t* __restrict__ rslot, int64_t n, int32_t slot) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (rslot[mid] < slot) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Movie.addRating (Movie.java:93-95), one thread per movie over its ratings in file order: the explicit
// roundings keep the compiler from contracting avg * n + score into one fused multiply-add
__global__ void sim_average_kernel(const int32_t* __restrict__ rslot, const float* __restrict__ score, int64_t n,
                                   int n_movies, double* __restrict__ avg, uint64_t* __restrict__ key,
                                   int32_t* __restrict__ iota) {
  SIM_GRID_STRIDE(m, n_movies) {
    const int64_t lo = lower_bound(rslot, n, (int32_t)m), hi = lower_bound(rslot, n, (int32_t)m + 1);
    double a = 0.0;
    for (int64_t k = lo; k < hi; ++k) {
      const double cnt = (double)(k - lo);
      a = __ddiv_rn(__dadd_rn(__dmul_rn(a, cnt), (double)score[k]), __dadd_rn(cnt, 1.0));
    }
    avg[m] = a;
    key[m] = desc_key(a);
    iota[m] = (int32_t)m;
  }
}

// One block per genre: the first kGenreTop movies of the by-rating order that carry genre g
__global__ void __launch_bounds__(kThreads)
sim_genre_top_kernel(const int32_t* __restrict__ order, const uint64_t* __restrict__ mask, int n_movies,
                     int32_t* __restrict__ glist, int32_t* __restrict__ gcnt) {
  using Scan = cub::BlockScan<int, kThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const int g = blockIdx.x;
  int base = 0;
  for (int i0 = 0; i0 < n_movies && base < kGenreTop; i0 += kThreads) {
    const int i = i0 + threadIdx.x;
    const int slot = i < n_movies ? order[i] : 0;
    const int flag = i < n_movies ? (int)((mask[slot] >> g) & 1ull) : 0;
    int pos, total;
    Scan(tmp).ExclusiveSum(flag, pos, total);
    if (flag && base + pos < kGenreTop) glist[g * kGenreTop + base + pos] = slot;
    base += total;                       // the same in every thread: the loop exits together
    __syncthreads();                     // tmp is reused
  }
  if (threadIdx.x == 0) gcnt[g] = base < kGenreTop ? base : kGenreTop;
}

// listed[slot] |= the bits of the genres whose first `top` entries hold it (an integer OR: the result does not
// depend on order)
__global__ void sim_listed_kernel(const int32_t* __restrict__ glist, const int32_t* __restrict__ gcnt, int n_genres,
                                  int top, unsigned long long* __restrict__ listed) {
  SIM_GRID_STRIDE(i, (int64_t)n_genres * kGenreTop) {
    const int g = (int)(i / kGenreTop), j = (int)(i % kGenreTop);
    if (j < gcnt[g] && j < top) atomicOr(listed + glist[i], 1ull << g);
  }
}

// HashMap.hash(Integer) = id ^ (id >>> 16); the bucket is its low bits.  iota[m] = m, the values of the sort
__global__ void sim_bucket_kernel(const int32_t* __restrict__ movie_id, int n, uint32_t cap_mask,
                                  uint32_t* __restrict__ bucket, int32_t* __restrict__ iota) {
  SIM_GRID_STRIDE(m, n) {
    const uint32_t h = (uint32_t)movie_id[m];
    bucket[m] = (h ^ (h >> 16)) & cap_mask;
    iota[m] = (int32_t)m;
  }
}

// getMovies' two sort keys along movieMap's order `hm`: Double.compare descending of the average, and
// Integer.compare descending of the release year (the sign bit flipped, then complemented)
__global__ void sim_global_keys_kernel(const int32_t* __restrict__ hm, const double* __restrict__ avg,
                                       const int32_t* __restrict__ year, int n, uint64_t* __restrict__ rkey,
                                       uint32_t* __restrict__ ykey) {
  SIM_GRID_STRIDE(i, n) {
    const int s = hm[i];
    rkey[i] = desc_key(avg[s]);
    if (year) ykey[i] = ~((uint32_t)year[s] ^ 0x80000000u);
  }
}

__global__ void sim_flag_kernel(const int32_t* __restrict__ list, int n, uint8_t* __restrict__ flag) {
  SIM_GRID_STRIDE(i, n) flag[list[i]] = 1;
}

// DataManager.loadMovieEmb sets each listed movie's vector in file order, so the last row of an id wins
__global__ void sim_emb_row_kernel(const int32_t* __restrict__ emb_id, int n_emb, const int32_t* __restrict__ ids,
                                   const int32_t* __restrict__ slots, int n_movies, int32_t* __restrict__ emb_row) {
  SIM_GRID_STRIDE(i, n_emb) {
    const int s = find_slot(ids, slots, n_movies, emb_id[i]);
    if (s >= 0) atomicMax(emb_row + s, (int32_t)i);
  }
}

struct QueryArgs {
  const int32_t *ids_sorted, *slot_sorted, *movie_id;
  const uint64_t *mask, *listed;
  const double* avg;
  const int32_t *glist, *gcnt;
  const float* emb;
  const int32_t* emb_row;
  int n_movies, dim;
  int np;                                // the sort width: a power of two >= every candidate list
  int width;                             // output entries per query on the device
  int emb_model;
  int top;                               // entries taken from each genre list
  int multi;                             // MULTIPLE: the two global lists follow the genres' segments
  const int32_t *rtop, *ytop;            // MULTIPLE: getMovies(100, "rating" / "releaseYear"), n_top entries each
  int n_top;
  const uint8_t* in_rtop;
};

constexpr uint64_t kPad = ~0ull;         // an empty sort entry: after every real one

__device__ __forceinline__ bool item_greater(const ulonglong2& a, const ulonglong2& b) {
  return a.x > b.x || (a.x == b.x && a.y > b.y);
}

// calculateSimilarScore (SimilarMovieProcess.java:145-159), each operation rounded once as Java does
__device__ __forceinline__ double default_score(uint64_t qmask, uint64_t cmask, double avg) {
  const int same = __popcll(qmask & cmask), sizes = __popcll(qmask) + __popcll(cmask);
  const double genre = __ddiv_rn(__ddiv_rn((double)same, (double)sizes), 2.0);
  return __dadd_rn(__dmul_rn(genre, 0.7), __dmul_rn(__ddiv_rn(avg, 5.0), 0.3));
}

// One block per query.  item[i] = (desc_key(score), (movie id ^ 2^31) << 32 | slot): ascending is the ranking.
__global__ void __launch_bounds__(kQueryThreads)
sim_query_kernel(QueryArgs a, const int32_t* __restrict__ query, int32_t* __restrict__ out_id,
                 double* __restrict__ out_score, int32_t* __restrict__ count, int32_t* __restrict__ status) {
  extern __shared__ ulonglong2 item[];
  __shared__ int s_gen[kMaxGenres + 2], s_off[kMaxGenres + 3], s_nseg;
  const int q = blockIdx.x, tid = threadIdx.x;
  const int slot = find_slot(a.ids_sorted, a.slot_sorted, a.n_movies, query[q]);
  const int qrow = slot >= 0 && a.emb_model ? a.emb_row[slot] : 0;
  if (slot < 0 || qrow < 0) {            // getRecList's empty list; the Java throws on a query without a vector
    if (tid == 0) {
      count[q] = 0;
      status[q] = slot < 0 ? SRS_SIMILAR_UNKNOWN_MOVIE : SRS_SIMILAR_NO_EMBEDDING;
    }
    return;
  }
  const uint64_t qmask = a.mask[slot];
  if (tid == 0) {                        // the query's genres ascending, and where each one's entries start
    int k = 0;
    s_off[0] = 0;
    for (uint64_t m = qmask; m; m &= m - 1, ++k) {
      s_gen[k] = __ffsll((long long)m) - 1;
      s_off[k + 1] = s_off[k] + min(a.gcnt[s_gen[k]], a.top);
    }
    if (a.multi) {                       // then getMovies(100, "rating") and getMovies(100, "releaseYear")
      s_gen[k] = kSegRating;
      s_off[k + 1] = s_off[k] + a.n_top;
      ++k;
      s_gen[k] = kSegYear;
      s_off[k + 1] = s_off[k] + a.n_top;
      ++k;
    }
    s_nseg = k;
  }
  __syncthreads();
  const int total = s_off[s_nseg];

  // candidateGenerator / multipleRetrievalCandidates: each (list, entry) once, kept where the candidate first
  // appears among the query's lists (a.listed marks the genres' lists, in_rtop the rating list)
  int kept = 0;
  for (int i0 = 0; i0 < a.np; i0 += kQueryThreads) {
    const int i = i0 + tid;
    ulonglong2 it = make_ulonglong2(kPad, kPad);
    if (i < total) {
      int k = 0;
      while (s_off[k + 1] <= i) ++k;
      const int g = s_gen[k], j = i - s_off[k];
      int c;
      uint64_t earlier;
      if (g >= 0) {
        c = a.glist[g * kGenreTop + j];
        earlier = a.listed[c] & qmask & ((1ull << g) - 1);
      } else if (g == kSegRating) {
        c = a.rtop[j];
        earlier = a.listed[c] & qmask;
      } else {
        c = a.ytop[j];
        earlier = (a.listed[c] & qmask) | a.in_rtop[c];
      }
      if (c != slot && earlier == 0)
        it = make_ulonglong2(0, ((uint64_t)((uint32_t)a.movie_id[c] ^ 0x80000000u) << 32) | (uint32_t)c);
    }
    if (i < a.np) item[i] = it;
    kept += __syncthreads_count(it.y != kPad);
  }

  // ranker: the scores
  if (!a.emb_model) {
    for (int i = tid; i < total; i += kQueryThreads)
      if (item[i].y != kPad) {
        const int c = (int)(uint32_t)item[i].y;
        item[i].x = desc_key(default_score(qmask, a.mask[c], a.avg[c]));
      }
  } else {
    const int warp = tid >> 5, lane = tid & 31;
    const float* qv = a.emb + (size_t)qrow * a.dim;
    for (int i = warp; i < total; i += kQueryThreads / 32) {
      if (item[i].y == kPad) continue;   // the same for the whole warp
      const int c = (int)(uint32_t)item[i].y;
      const int r = a.emb_row[c];
      double s = -1.0;                   // Embedding.calculateSimilarity of a missing vector
      if (r >= 0) {
        double dot, n1, n2;
        cosine_sums(qv, a.emb + (size_t)r * a.dim, a.dim, lane, dot, n1, n2);
        s = cosine_value(dot, n1, n2);
      }
      if (lane == 0) item[i].x = desc_key(s);
    }
  }
  __syncthreads();

  // bitonic sort of item[0 .. np), ascending
  for (int w = 2; w <= a.np; w <<= 1)
    for (int j = w >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < a.np / 2; t += kQueryThreads) {
        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1)), hi = lo | j;
        const ulonglong2 x = item[lo], y = item[hi];
        if (item_greater(x, y) == ((lo & w) == 0)) {
          item[lo] = y;
          item[hi] = x;
        }
      }
      __syncthreads();
    }

  const int n_out = kept < a.width ? kept : a.width;
  for (int r = tid; r < n_out; r += kQueryThreads) {
    out_id[(size_t)q * a.width + r] = (int32_t)((uint32_t)(item[r].y >> 32) ^ 0x80000000u);
    out_score[(size_t)q * a.width + r] = key_score(item[r].x);
  }
  if (tid == 0) {
    count[q] = n_out;
    status[q] = SRS_SIMILAR_OK;
  }
}

struct RecallArgs {
  const int32_t *ids_sorted, *slot_sorted, *movie_id, *emb_row;
  const int32_t* pool;                   // [n_pool] slots in ascending movie id
  const float* emb;
  int n_movies, dim, n_pool;
  int width;                             // output entries per query on the device
};

// retrievalCandidatesByEmbedding, one block per query: the cosine of every pool movie (one warp each, as the emb
// ranker), then a stable block radix sort of (~desc_key(score), pool index) - Double.compare ascending, NaN last,
// and ties in pool order, which is movie id order.  The scores are staged in the sort's own storage.
template <int kT, int kItems>
__global__ void __launch_bounds__(kT)
sim_emb_recall_kernel(RecallArgs a, const int32_t* __restrict__ query, int32_t* __restrict__ out_id,
                      double* __restrict__ out_score, int32_t* __restrict__ count, int32_t* __restrict__ status) {
  using Sort = cub::BlockRadixSort<uint64_t, kT, kItems, uint16_t>;
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* key = reinterpret_cast<uint64_t*>(smem);
  auto& tmp = *reinterpret_cast<typename Sort::TempStorage*>(smem);
  const int q = blockIdx.x, tid = threadIdx.x;
  const int slot = find_slot(a.ids_sorted, a.slot_sorted, a.n_movies, query[q]);
  const int qrow = slot >= 0 ? a.emb_row[slot] : -1;
  if (slot < 0 || qrow < 0) {            // the Java returns null for both
    if (tid == 0) {
      count[q] = 0;
      status[q] = slot < 0 ? SRS_SIMILAR_UNKNOWN_MOVIE : SRS_SIMILAR_NO_EMBEDDING;
    }
    return;
  }
  const int warp = tid >> 5, lane = tid & 31;
  const float* qv = a.emb + (size_t)qrow * a.dim;
  for (int j = warp; j < a.n_pool; j += kT / 32) {
    const int r = a.emb_row[a.pool[j]];
    double s = -1.0;                     // calculateEmbSimilarScore of a candidate without a vector
    if (r >= 0) {
      double dot, n1, n2;
      cosine_sums(qv, a.emb + (size_t)r * a.dim, a.dim, lane, dot, n1, n2);
      s = cosine_value(dot, n1, n2);
    }
    if (lane == 0) key[j] = ~desc_key(s);
  }
  __syncthreads();
  uint64_t k[kItems];
  uint16_t v[kItems];
#pragma unroll
  for (int i = 0; i < kItems; ++i) {     // padding sorts after every entry: ~0 ties only NaN, and comes later
    const int j = tid * kItems + i;
    k[i] = j < a.n_pool ? key[j] : ~0ull;
    v[i] = (uint16_t)j;
  }
  __syncthreads();                       // key[] and tmp share the storage
  Sort(tmp).Sort(k, v);
  const int n_out = a.n_pool < a.width ? a.n_pool : a.width;
#pragma unroll
  for (int i = 0; i < kItems; ++i) {
    const int r = tid * kItems + i;
    if (r < n_out) {
      out_id[(size_t)q * a.width + r] = a.movie_id[a.pool[v[i]]];
      out_score[(size_t)q * a.width + r] = key_score(~k[i]);
    }
  }
  if (tid == 0) {
    count[q] = n_out;
    status[q] = SRS_SIMILAR_OK;
  }
}

// the two instantiations: a small catalogue's pool, and getMovies(10000, ...)'s
constexpr int kRecallSmallT = 128, kRecallSmallItems = 8;
constexpr int kRecallT = 512, kRecallItems = 20;
static_assert(kRecallT * kRecallItems >= kPool && kPool <= 65536, "the pool fits one block's sort and a uint16");

// java.util.HashMap<Integer, Movie>'s table length once DataManager.loadMovieData has put ids[0 .. n) in load
// order (putVal, resize and treeifyBin of JDK 8 on): 16 at the first put, doubled when the size passes 3/4 of it,
// or when a put makes a bin's ninth entry while the table is shorter than MIN_TREEIFY_CAPACITY (64).  0 when such a
// put meets a table of 64 or more: that bin becomes a tree, and its iteration order is no longer load order.
int64_t hashmap_capacity(const int32_t* ids, int32_t n) {
  auto spread = [](int32_t id) { const uint32_t h = (uint32_t)id; return h ^ (h >> 16); };
  int64_t cap = 16;
  std::vector<int32_t> bin(cap, 0);
  auto rebin = [&](int32_t upto) {
    bin.assign(cap, 0);
    for (int32_t i = 0; i < upto; ++i) ++bin[spread(ids[i]) & (cap - 1)];
  };
  for (int32_t i = 0; i < n; ++i) {
    if (++bin[spread(ids[i]) & (cap - 1)] > 8) {          // TREEIFY_THRESHOLD
      if (cap >= 64) return 0;
      cap <<= 1;
      rebin(i + 1);
    }
    if (i + 1 > cap / 4 * 3) {
      cap <<= 1;
      rebin(i + 1);
    }
  }
  return cap;
}

int bits_for(int64_t n) {                // radix bits covering 0 .. n
  int b = 1;
  while (b < 63 && (int64_t(1) << b) <= n) ++b;
  return b;
}

template <class T>
int persist(T** p, size_t count) {       // a catalogue allocation, freed by its destructor
  CUDA_TRY(cudaMalloc(p, (count ? count : 1) * sizeof(T)));
  return SRS_OK;
}

int create(const int32_t* movie_id, int32_t n_movies, const int32_t* genre_off, const int32_t* genre,
           int32_t n_genres, const int32_t* rating_movie, const float* rating_score, int64_t n_ratings,
           const int32_t* emb_id, const float* emb, int32_t n_emb, int32_t dim, const int32_t* release_year,
           int32_t device, srs_similar_catalog** out) {
  if (!out) return failf(SRS_ERR_INVALID, "similar catalog: null output handle");
  *out = nullptr;
  if (n_movies < 0) return failf(SRS_ERR_INVALID, "similar catalog: n_movies %d < 0", n_movies);
  if (n_genres < 0 || n_genres > kMaxGenres)
    return failf(SRS_ERR_INVALID, "similar catalog: %d genres; 0 .. %d are supported", n_genres, kMaxGenres);
  if (n_movies > 0 && (!movie_id || !genre_off))
    return failf(SRS_ERR_INVALID, "similar catalog: null movie_id or genre_off");
  if (n_movies > 0 && genre_off[0] != 0) return failf(SRS_ERR_INVALID, "similar catalog: genre_off[0] != 0");
  std::vector<uint64_t> mask(n_movies);
  for (int32_t m = 0; m < n_movies; ++m) {
    if (genre_off[m + 1] < genre_off[m])
      return failf(SRS_ERR_INVALID, "similar catalog: genre_off decreases at movie %d", m);
    for (int32_t k = genre_off[m]; k < genre_off[m + 1]; ++k) {
      if (!genre) return failf(SRS_ERR_INVALID, "similar catalog: null genre");
      const int32_t g = genre[k];
      if (g < 0 || g >= n_genres)
        return failf(SRS_ERR_INVALID, "similar catalog: movie %d: genre %d outside 0 .. %d", movie_id[m], g,
                     n_genres - 1);
      if (mask[m] >> g & 1)
        return failf(SRS_ERR_INVALID, "similar catalog: movie %d lists genre %d twice", movie_id[m], g);
      mask[m] |= 1ull << g;
    }
  }
  {
    std::vector<int32_t> ids(movie_id, movie_id + n_movies);
    std::sort(ids.begin(), ids.end());
    const auto dup = std::adjacent_find(ids.begin(), ids.end());
    if (dup != ids.end()) return failf(SRS_ERR_INVALID, "similar catalog: movie id %d appears twice", *dup);
  }
  if (n_ratings < 0 || n_ratings > INT32_MAX)
    return failf(SRS_ERR_INVALID, "similar catalog: n_ratings %lld outside 0 .. 2^31 - 1", (long long)n_ratings);
  if (n_ratings > 0 && (!rating_movie || !rating_score))
    return failf(SRS_ERR_INVALID, "similar catalog: null rating_movie or rating_score");
  if (n_emb < 0 || dim < 0) return failf(SRS_ERR_INVALID, "similar catalog: n_emb %d or dim %d < 0", n_emb, dim);
  if (n_emb > 0 && (dim < 1 || !emb_id || !emb))
    return failf(SRS_ERR_INVALID, "similar catalog: %d vectors need dim >= 1 (got %d), emb_id and emb", n_emb, dim);
  const int64_t cap = hashmap_capacity(movie_id, n_movies);

  HostCall c;
  PROPAGATE(c.begin(device));
  srs_similar_catalog* h = new (std::nothrow) srs_similar_catalog;
  if (!h) return failf(SRS_ERR_NOMEM, "similar catalog: out of host memory");
  std::unique_ptr<srs_similar_catalog> owner(h);
  h->device = device;
  h->n_movies = n_movies;
  h->n_genres = n_genres;
  h->dim = n_emb > 0 ? dim : 0;
  h->hash_order = cap > 0;
  h->has_year = release_year != nullptr;
  const int nm = n_movies;
  const int64_t nr = n_ratings;

  // the movies: id -> slot, and their genres
  int32_t *d_ids, *d_iota;
  PROPAGATE(c.upload(&d_ids, movie_id, nm));
  CUDA_TRY(c.sc.alloc(&d_iota, nm));
  PROPAGATE(persist(&h->ids_sorted, nm));
  PROPAGATE(persist(&h->slot_sorted, nm));
  PROPAGATE(persist(&h->movie_id, nm));
  PROPAGATE(persist(&h->mask, nm));
  PROPAGATE(persist(&h->listed, nm));
  PROPAGATE(persist(&h->avg, nm));
  PROPAGATE(persist(&h->glist, (size_t)n_genres * kGenreTop));
  PROPAGATE(persist(&h->gcnt, n_genres));
  PROPAGATE(persist(&h->emb_row, nm));
  PROPAGATE(persist(&h->listed_multi, nm));
  PROPAGATE(persist(&h->in_rtop, nm));
  if (nm) {
    CUDA_TRY(cudaMemcpyAsync(h->movie_id, d_ids, sizeof(int32_t) * nm, cudaMemcpyDeviceToDevice, c.s));
    CUDA_TRY(cudaMemcpyAsync(h->mask, mask.data(), sizeof(uint64_t) * nm, cudaMemcpyHostToDevice, c.s));
    sim_iota_kernel<<<grid_for(nm, kThreads), kThreads, 0, c.s>>>(d_iota, nm);
    LAUNCHED();
    CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_ids, h->ids_sorted, d_iota, h->slot_sorted, nm, 0, 32,
                                               c.s));
  }

  // Movie.averageRating: each movie's ratings in file order
  int32_t *d_rmovie, *d_rslot, *d_rslot_sorted;
  float *d_score, *d_score_sorted;
  PROPAGATE(c.upload(&d_rmovie, rating_movie, (size_t)nr));
  PROPAGATE(c.upload(&d_score, rating_score, (size_t)nr));
  CUDA_TRY(c.sc.alloc(&d_rslot, (size_t)nr));
  CUDA_TRY(c.sc.alloc(&d_rslot_sorted, (size_t)nr));
  CUDA_TRY(c.sc.alloc(&d_score_sorted, (size_t)nr));
  if (nr) {
    sim_rating_slot_kernel<<<grid_for(nr, kThreads), kThreads, 0, c.s>>>(d_rmovie, nr, h->ids_sorted,
                                                                         h->slot_sorted, nm, d_rslot);
    LAUNCHED();
    CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_rslot, d_rslot_sorted, d_score, d_score_sorted,
                                               (int)nr, 0, bits_for(nm), c.s));
  }
  uint64_t *d_key, *d_key_sorted;
  int32_t* d_order;
  CUDA_TRY(c.sc.alloc(&d_key, nm));
  CUDA_TRY(c.sc.alloc(&d_key_sorted, nm));
  CUDA_TRY(c.sc.alloc(&d_order, nm));
  if (nm) {
    sim_average_kernel<<<grid_for(nm, kThreads), kThreads, 0, c.s>>>(d_rslot_sorted, d_score_sorted, nr, nm, h->avg,
                                                                     d_key, d_iota);
    LAUNCHED();
    // getMoviesByGenre's order for every genre at once: the stable sort keeps load order among equal averages
    CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_key, d_key_sorted, d_iota, d_order, nm, 0, 64, c.s));
  }
  std::vector<int32_t> gcnt(n_genres, 0);
  CUDA_TRY(cudaMemsetAsync(h->listed, 0, sizeof(uint64_t) * (nm ? nm : 1), c.s));
  CUDA_TRY(cudaMemsetAsync(h->listed_multi, 0, sizeof(uint64_t) * (nm ? nm : 1), c.s));
  if (n_genres) {
    if (nm) {
      sim_genre_top_kernel<<<n_genres, kThreads, 0, c.s>>>(d_order, h->mask, nm, h->glist, h->gcnt);
      LAUNCHED();
      sim_listed_kernel<<<grid_for((int64_t)n_genres * kGenreTop, kThreads), kThreads, 0, c.s>>>(
          h->glist, h->gcnt, n_genres, kGenreTop, reinterpret_cast<unsigned long long*>(h->listed));
      LAUNCHED();
      sim_listed_kernel<<<grid_for((int64_t)n_genres * kGenreTop, kThreads), kThreads, 0, c.s>>>(
          h->glist, h->gcnt, n_genres, kMultiGenreTop, reinterpret_cast<unsigned long long*>(h->listed_multi));
      LAUNCHED();
    } else {
      CUDA_TRY(cudaMemsetAsync(h->gcnt, 0, sizeof(int32_t) * n_genres, c.s));
    }
    CUDA_TRY(cudaMemcpyAsync(gcnt.data(), h->gcnt, sizeof(int32_t) * n_genres, cudaMemcpyDeviceToHost, c.s));
  }

  // getMovies(size, sortBy): stable sorts of movieMap's iteration order - by bucket, load order within one
  CUDA_TRY(cudaMemsetAsync(h->in_rtop, 0, nm ? nm : 1, c.s));
  std::vector<int32_t> pool;
  if (nm && h->hash_order) {
    h->n_pool = std::min(nm, kPool);
    h->n_rec = std::min(nm, kRecForYou);
    h->n_top = h->has_year ? std::min(nm, kGlobalTop) : 0;
    uint32_t *d_bucket, *d_bucket_sorted, *d_ykey = nullptr, *d_ykey_sorted = nullptr;
    int32_t *d_slot, *d_hm, *d_rorder, *d_year = nullptr, *d_yorder = nullptr;
    uint64_t *d_rkey, *d_rkey_sorted;
    CUDA_TRY(c.sc.alloc(&d_bucket, nm));
    CUDA_TRY(c.sc.alloc(&d_bucket_sorted, nm));
    CUDA_TRY(c.sc.alloc(&d_slot, nm));
    CUDA_TRY(c.sc.alloc(&d_hm, nm));
    CUDA_TRY(c.sc.alloc(&d_rkey, nm));
    CUDA_TRY(c.sc.alloc(&d_rkey_sorted, nm));
    CUDA_TRY(c.sc.alloc(&d_rorder, nm));
    if (h->has_year) {
      PROPAGATE(c.upload(&d_year, release_year, nm));
      CUDA_TRY(c.sc.alloc(&d_ykey, nm));
      CUDA_TRY(c.sc.alloc(&d_ykey_sorted, nm));
      CUDA_TRY(c.sc.alloc(&d_yorder, nm));
    }
    sim_bucket_kernel<<<grid_for(nm, kThreads), kThreads, 0, c.s>>>(h->movie_id, nm, (uint32_t)(cap - 1), d_bucket,
                                                                      d_slot);
    LAUNCHED();
    CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_bucket, d_bucket_sorted, d_slot, d_hm, nm, 0,
                                               bits_for(cap - 1), c.s));
    sim_global_keys_kernel<<<grid_for(nm, kThreads), kThreads, 0, c.s>>>(d_hm, h->avg, d_year, nm, d_rkey, d_ykey);
    LAUNCHED();
    CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_rkey, d_rkey_sorted, d_hm, d_rorder, nm, 0, 64, c.s));
    PROPAGATE(persist(&h->pool, h->n_pool));
    PROPAGATE(persist(&h->rec, h->n_rec));
    CUDA_TRY(cudaMemcpyAsync(h->rec, d_rorder, sizeof(int32_t) * h->n_rec, cudaMemcpyDeviceToDevice, c.s));
    pool.resize(h->n_pool);
    CUDA_TRY(cudaMemcpyAsync(pool.data(), d_rorder, sizeof(int32_t) * h->n_pool, cudaMemcpyDeviceToHost, c.s));
    if (h->has_year) {
      CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_ykey, d_ykey_sorted, d_hm, d_yorder, nm, 0, 32,
                                                 c.s));
      PROPAGATE(persist(&h->rtop, h->n_top));
      PROPAGATE(persist(&h->ytop, h->n_top));
      CUDA_TRY(cudaMemcpyAsync(h->rtop, d_rorder, sizeof(int32_t) * h->n_top, cudaMemcpyDeviceToDevice, c.s));
      CUDA_TRY(cudaMemcpyAsync(h->ytop, d_yorder, sizeof(int32_t) * h->n_top, cudaMemcpyDeviceToDevice, c.s));
      sim_flag_kernel<<<grid_for(h->n_top, kThreads), kThreads, 0, c.s>>>(h->rtop, h->n_top, h->in_rtop);
      LAUNCHED();
    }
  }

  // the vectors
  CUDA_TRY(cudaMemsetAsync(h->emb_row, 0xFF, sizeof(int32_t) * (nm ? nm : 1), c.s));
  if (n_emb > 0) {
    CUDA_TRY(cudaMalloc(&h->emb, sizeof(float) * (size_t)n_emb * dim));
    CUDA_TRY(cudaMemcpyAsync(h->emb, emb, sizeof(float) * (size_t)n_emb * dim, cudaMemcpyHostToDevice, c.s));
    int32_t* d_eid;
    PROPAGATE(c.upload(&d_eid, emb_id, n_emb));
    if (nm) {
      sim_emb_row_kernel<<<grid_for(n_emb, kThreads), kThreads, 0, c.s>>>(d_eid, n_emb, h->ids_sorted,
                                                                          h->slot_sorted, nm, h->emb_row);
      LAUNCHED();
    }
  }
  CUDA_TRY(cudaStreamSynchronize(c.s));
  for (int32_t m = 0; m < nm; ++m) {
    int32_t s = 0;
    for (uint64_t b = mask[m]; b; b &= b - 1) s += gcnt[__builtin_ctzll(b)];
    h->max_cands = std::max(h->max_cands, s);
    int32_t sm = 2 * h->n_top;
    for (uint64_t b = mask[m]; b; b &= b - 1) sm += std::min(gcnt[__builtin_ctzll(b)], kMultiGenreTop);
    h->max_multi = std::max(h->max_multi, sm);
  }
  // the embedding pool in movie id order, so that the recall's stable sort leaves tied scores by id
  std::sort(pool.begin(), pool.end(), [&](int32_t x, int32_t y) { return movie_id[x] < movie_id[y]; });
  if (!pool.empty())
    CUDA_TRY(cudaMemcpy(h->pool, pool.data(), sizeof(int32_t) * pool.size(), cudaMemcpyHostToDevice));
  *out = owner.release();
  return SRS_OK;
}

int query(const srs_similar_catalog* h, int32_t candidates, const int32_t* movie_ids, int32_t n_queries, int32_t size,
          int32_t model, int32_t* out_ids, double* out_scores, int32_t* out_count, int32_t* out_status) {
  if (n_queries < 0) return failf(SRS_ERR_INVALID, "similar movies: n_queries %d < 0", n_queries);
  if (size < 1) return failf(SRS_ERR_INVALID, "similar movies: size %d < 1", size);
  if (model != SRS_SIMILAR_DEFAULT && model != SRS_SIMILAR_EMB)
    return failf(SRS_ERR_INVALID, "similar movies: unknown model %d", model);
  if (candidates != SRS_SIMILAR_CANDIDATES_GENRE && candidates != SRS_SIMILAR_CANDIDATES_MULTIPLE)
    return failf(SRS_ERR_INVALID, "similar movies: unknown candidate source %d", candidates);
  if (!h) return failf(SRS_ERR_INVALID, "similar movies: null catalog");
  const bool multi = candidates == SRS_SIMILAR_CANDIDATES_MULTIPLE;
  if (multi && !h->has_year)
    return failf(SRS_ERR_INVALID, "similar movies: multi-channel recall needs a catalogue created with release years");
  if (multi && !h->hash_order)
    return failf(SRS_ERR_INVALID, "similar movies: a HashMap bin of the movie ids is treeified (9 or more ids in one "
                 "bucket of a table of 64 or more), so getMovies' order of ties is not load order within a bucket");
  if (n_queries > 0 && (!movie_ids || !out_ids || !out_scores || !out_count || !out_status))
    return failf(SRS_ERR_INVALID, "similar movies: null query or output array");
  if (n_queries == 0) return SRS_OK;
  const size_t Q = (size_t)n_queries;
  memset(out_ids, 0, sizeof(int32_t) * Q * size);
  memset(out_scores, 0, sizeof(double) * Q * size);

  const int max_cands = multi ? h->max_multi : h->max_cands;
  int np = 32;
  while (np < max_cands) np <<= 1;
  const int width = std::max(1, std::min(size, max_cands));
  HostCall c;
  PROPAGATE(c.begin(h->device));
  int32_t *d_query, *d_ids, *d_count, *d_status;
  double* d_scores;
  PROPAGATE(c.upload(&d_query, movie_ids, Q));
  CUDA_TRY(c.sc.alloc(&d_ids, Q * width));
  CUDA_TRY(c.sc.alloc(&d_scores, Q * width));
  CUDA_TRY(c.sc.alloc(&d_count, Q));
  CUDA_TRY(c.sc.alloc(&d_status, Q));
  CUDA_TRY(cudaMemsetAsync(d_ids, 0, sizeof(int32_t) * Q * width, c.s));
  CUDA_TRY(cudaMemsetAsync(d_scores, 0, sizeof(double) * Q * width, c.s));
  const QueryArgs a{h->ids_sorted, h->slot_sorted, h->movie_id, h->mask, multi ? h->listed_multi : h->listed, h->avg,
                    h->glist, h->gcnt, h->emb, h->emb_row, h->n_movies, h->dim, np, width, model == SRS_SIMILAR_EMB,
                    multi ? kMultiGenreTop : kGenreTop, multi, h->rtop, h->ytop, multi ? h->n_top : 0, h->in_rtop};
  const size_t smem = sizeof(ulonglong2) * np;
  CUDA_TRY(cudaFuncSetAttribute(sim_query_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sim_query_kernel<<<n_queries, kQueryThreads, smem, c.s>>>(a, d_query, d_ids, d_scores, d_count, d_status);
  LAUNCHED();
  CUDA_TRY(cudaMemcpy2DAsync(out_ids, sizeof(int32_t) * size, d_ids, sizeof(int32_t) * width,
                             sizeof(int32_t) * width, Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpy2DAsync(out_scores, sizeof(double) * size, d_scores, sizeof(double) * width,
                             sizeof(double) * width, Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(out_count, d_count, sizeof(int32_t) * Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(out_status, d_status, sizeof(int32_t) * Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));
  return SRS_OK;
}

template <int kT, int kItems>
int launch_recall(const RecallArgs& a, int n_queries, cudaStream_t s, const int32_t* query, int32_t* ids,
                  double* scores, int32_t* count, int32_t* status) {
  using Sort = cub::BlockRadixSort<uint64_t, kT, kItems, uint16_t>;
  const size_t smem = std::max(sizeof(typename Sort::TempStorage), sizeof(uint64_t) * a.n_pool);
  CUDA_TRY(cudaFuncSetAttribute(sim_emb_recall_kernel<kT, kItems>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)smem));
  sim_emb_recall_kernel<kT, kItems><<<n_queries, kT, smem, s>>>(a, query, ids, scores, count, status);
  LAUNCHED();
  return SRS_OK;
}

int recall(const srs_similar_catalog* h, const int32_t* movie_ids, int32_t n_queries, int32_t size, int32_t* out_ids,
           double* out_scores, int32_t* out_count, int32_t* out_status) {
  if (n_queries < 0) return failf(SRS_ERR_INVALID, "embedding recall: n_queries %d < 0", n_queries);
  if (size < 1) return failf(SRS_ERR_INVALID, "embedding recall: size %d < 1", size);
  if (!h) return failf(SRS_ERR_INVALID, "embedding recall: null catalog");
  if (!h->hash_order)
    return failf(SRS_ERR_INVALID, "embedding recall: a HashMap bin of the movie ids is treeified (9 or more ids in "
                 "one bucket of a table of 64 or more), so getMovies' order of ties is not load order within a bucket");
  if (n_queries > 0 && (!movie_ids || !out_ids || !out_scores || !out_count || !out_status))
    return failf(SRS_ERR_INVALID, "embedding recall: null query or output array");
  if (n_queries == 0) return SRS_OK;
  const size_t Q = (size_t)n_queries;
  memset(out_ids, 0, sizeof(int32_t) * Q * size);
  memset(out_scores, 0, sizeof(double) * Q * size);

  const int width = std::max(1, std::min(size, h->n_pool));
  HostCall c;
  PROPAGATE(c.begin(h->device));
  int32_t *d_query, *d_ids, *d_count, *d_status;
  double* d_scores;
  PROPAGATE(c.upload(&d_query, movie_ids, Q));
  CUDA_TRY(c.sc.alloc(&d_ids, Q * width));
  CUDA_TRY(c.sc.alloc(&d_scores, Q * width));
  CUDA_TRY(c.sc.alloc(&d_count, Q));
  CUDA_TRY(c.sc.alloc(&d_status, Q));
  CUDA_TRY(cudaMemsetAsync(d_ids, 0, sizeof(int32_t) * Q * width, c.s));
  CUDA_TRY(cudaMemsetAsync(d_scores, 0, sizeof(double) * Q * width, c.s));
  const RecallArgs a{h->ids_sorted, h->slot_sorted, h->movie_id, h->emb_row, h->pool, h->emb, h->n_movies, h->dim,
                     h->n_pool, width};
  if (h->n_pool <= kRecallSmallT * kRecallSmallItems)
    PROPAGATE((launch_recall<kRecallSmallT, kRecallSmallItems>(a, n_queries, c.s, d_query, d_ids, d_scores, d_count,
                                                                d_status)));
  else
    PROPAGATE((launch_recall<kRecallT, kRecallItems>(a, n_queries, c.s, d_query, d_ids, d_scores, d_count,
                                                      d_status)));
  CUDA_TRY(cudaMemcpy2DAsync(out_ids, sizeof(int32_t) * size, d_ids, sizeof(int32_t) * width,
                             sizeof(int32_t) * width, Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpy2DAsync(out_scores, sizeof(double) * size, d_scores, sizeof(double) * width,
                             sizeof(double) * width, Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(out_count, d_count, sizeof(int32_t) * Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(out_status, d_status, sizeof(int32_t) * Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));
  return SRS_OK;
}

}  // namespace

SimilarCatalogView similar_catalog_view(const srs_similar_catalog* h) {
  return {h->device, h->n_movies, h->dim, h->hash_order, h->movie_id, h->emb, h->emb_row, h->n_rec, h->rec};
}

}  // namespace srs

extern "C" int srs_similar_catalog_create_host(const int32_t* movie_id, int32_t n_movies, const int32_t* genre_off,
                                               const int32_t* genre, int32_t n_genres, const int32_t* rating_movie,
                                               const float* rating_score, int64_t n_ratings, const int32_t* emb_id,
                                               const float* emb, int32_t n_emb, int32_t dim, int32_t device,
                                               srs_similar_catalog** out) {
  return srs::create(movie_id, n_movies, genre_off, genre, n_genres, rating_movie, rating_score, n_ratings, emb_id,
                     emb, n_emb, dim, nullptr, device, out);
}

extern "C" int srs_similar_catalog_create_ex_host(const int32_t* movie_id, int32_t n_movies,
                                                  const int32_t* genre_off, const int32_t* genre, int32_t n_genres,
                                                  const int32_t* rating_movie, const float* rating_score,
                                                  int64_t n_ratings, const int32_t* emb_id, const float* emb,
                                                  int32_t n_emb, int32_t dim, const int32_t* release_year,
                                                  int32_t device, srs_similar_catalog** out) {
  return srs::create(movie_id, n_movies, genre_off, genre, n_genres, rating_movie, rating_score, n_ratings, emb_id,
                     emb, n_emb, dim, release_year, device, out);
}

extern "C" int srs_similar_movies_host(const srs_similar_catalog* catalog, const int32_t* movie_ids,
                                       int32_t n_queries, int32_t size, int32_t model, int32_t* out_ids,
                                       double* out_scores, int32_t* out_count, int32_t* out_status) {
  return srs::query(catalog, SRS_SIMILAR_CANDIDATES_GENRE, movie_ids, n_queries, size, model, out_ids, out_scores,
                    out_count, out_status);
}

extern "C" int srs_similar_movies_candidates_host(const srs_similar_catalog* catalog, int32_t candidates,
                                                  const int32_t* movie_ids, int32_t n_queries, int32_t size,
                                                  int32_t model, int32_t* out_ids, double* out_scores,
                                                  int32_t* out_count, int32_t* out_status) {
  return srs::query(catalog, candidates, movie_ids, n_queries, size, model, out_ids, out_scores, out_count,
                    out_status);
}

extern "C" int srs_similar_embedding_recall_host(const srs_similar_catalog* catalog, const int32_t* movie_ids,
                                                 int32_t n_queries, int32_t size, int32_t* out_ids,
                                                 double* out_scores, int32_t* out_count, int32_t* out_status) {
  return srs::recall(catalog, movie_ids, n_queries, size, out_ids, out_scores, out_count, out_status);
}

extern "C" void srs_similar_catalog_destroy(srs_similar_catalog* catalog) { delete catalog; }
