// graphemb.cu - the reference's DeepWalk graph embedding (Embedding.scala:140-228, 254-266) on one device: the item
// transition matrix of consecutive positive ratings, random walks over it, and Word2Vec over the walks.  DESIGN.md
// section 4.14 gives the semantics and the orders Scala leaves open.
//
// One stream, after i2v_positive_corpus (item2vec.cu) has built the sentences:
//   1. ge_pair_kernel                   a 49-bit key (a << 24 | b) per consecutive pair of a sentence, a sentinel
//                                       (bit 48) elsewhere;
//   2. DeviceRadixSort + RunLengthEncode the distinct pairs by (source, target) ascending, with their counts;
//   3. ge_row_flag_kernel + select      the first pair of each source: a CSR by source;
//   4. ge_row_kernel                    one thread per source: out(a), P(a->b) = count / out(a) and the row's
//                                       cumulative sums, added left to right in double;
//   5. ge_dist_kernel                   one thread: dist(a) = out(a) / pairTotal and its cumulative sums, likewise;
//   6. ge_walk_kernel                   one thread per walk, each draw a binary search of a cumulative row.
// srs_graph_embedding_host then flattens the walks (ge_flat_kernel + two selects) into words keyed by walk and
// hands them to word2vec_fit (item2vec.cu).  Integer atomics only in the counting; every double sum has one fixed
// order, so the same inputs give the same bits.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <vector>

#include "../../include/srs_ctr.h"
#include "kernels.h"

namespace srs {
namespace {

constexpr int64_t kMaxWalkWords = 21000000;   // num_walks * walk_length: item2vec's bound on the corpus
constexpr uint64_t kSentinel = 1ull << 48;
constexpr uint32_t kIdMask = (1u << 24) - 1;

int ge_fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  return set_last_error(code, buf);
}

#define GE_TRY(expr)                                                                                      \
  do {                                                                                                    \
    cudaError_t e__ = (expr);                                                                             \
    if (e__ != cudaSuccess)                                                                               \
      return ge_fail(SRS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

#define GE_LAUNCHED()                                                                                     \
  do {                                                                                                    \
    ++g_launch_count;                                                                                     \
    GE_TRY(cudaGetLastError());                                                                           \
  } while (0)

// item2vec.cu's counter-based hash: splitmix64's finaliser of x + (i + 1) * golden
__host__ __device__ __forceinline__ uint64_t splitmix(uint64_t x, uint64_t i) {
  uint64_t z = x + (i + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

int grid_for(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  return (int)(b < 1 ? 1 : b > 132 * 64 ? 132 * 64 : b);
}

struct StreamGuard {
  cudaStream_t s = nullptr;
  ~StreamGuard() {
    if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
  }
};

__global__ void ge_pair_kernel(const int32_t* __restrict__ movie, const uint32_t* __restrict__ user,
                               const int* __restrict__ n_pos, int n, uint64_t* __restrict__ key,
                               int32_t* __restrict__ iota) {
  const int np = *n_pos;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const bool pair = i + 1 < np && user[i] == user[i + 1];
    key[i] = pair ? ((uint64_t)(uint32_t)movie[i] << 24) | (uint32_t)movie[i + 1] : kSentinel;
    iota[i] = i;
  }
}

// the number of runs that are pairs: the sorted sentinels, if any, make the last run
__device__ __forceinline__ int pair_runs(const uint64_t* ukey, const int* n_runs) {
  int ne = *n_runs;
  if (ne && (ukey[ne - 1] & kSentinel)) --ne;
  return ne;
}

__global__ void ge_row_flag_kernel(const uint64_t* __restrict__ ukey, const int* __restrict__ n_runs, int n,
                                   uint8_t* __restrict__ flag) {
  const int ne = pair_runs(ukey, n_runs);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    flag[i] = i < ne && (i == 0 || (ukey[i] >> 24) != (ukey[i - 1] >> 24));
}

struct Transitions {                  // device
  int32_t* source;                    // [S] ascending
  int32_t* row_ptr;                   // [S + 1]
  int32_t* out;                       // [S] out(a)
  double* dist;                       // [S] out(a) / pairTotal
  double* cdf;                        // [S] its cumulative sums
  int32_t* target;                    // [E] ascending within a row
  int32_t* count;                     // [E]
  double* prob;                       // [E] count / out(a)
  double* cum;                        // [E] the row's cumulative sums
  int32_t* row_of;                    // [n_slots] row of a movie id, -1 if it has no outgoing pair
  int* n_rows;                        // [2] S, E
};

__global__ void ge_row_kernel(const uint64_t* __restrict__ ukey, const int32_t* __restrict__ runs,
                              const int* __restrict__ n_runs, const int32_t* __restrict__ row_start, Transitions t) {
  const int S = t.n_rows[0];
  const int ne = pair_runs(ukey, n_runs);
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < S; r += gridDim.x * blockDim.x) {
    const int lo = row_start[r], hi = r + 1 < S ? row_start[r + 1] : ne;
    int out = 0;
    for (int e = lo; e < hi; ++e) out += runs[e];
    double cum = 0.0;
    for (int e = lo; e < hi; ++e) {
      const double p = __ddiv_rn((double)runs[e], (double)out);
      cum = __dadd_rn(cum, p);
      t.target[e] = (int32_t)(ukey[e] & kIdMask);
      t.count[e] = runs[e];
      t.prob[e] = p;
      t.cum[e] = cum;
    }
    const int a = (int)(ukey[lo] >> 24);
    t.source[r] = a;
    t.row_ptr[r] = lo;
    t.out[r] = out;
    t.row_of[a] = r;
  }
}

// one thread: pairTotal, the source distribution and its cumulative sums in ascending source order
__global__ void ge_dist_kernel(const uint64_t* __restrict__ ukey, const int* __restrict__ n_runs, Transitions t) {
  if (blockIdx.x | threadIdx.x) return;
  const int S = t.n_rows[0];
  const int ne = pair_runs(ukey, n_runs);
  t.row_ptr[S] = ne;
  t.n_rows[1] = ne;
  int64_t total = 0;
  for (int r = 0; r < S; ++r) total += t.out[r];
  double cdf = 0.0;
  for (int r = 0; r < S; ++r) {
    const double d = __ddiv_rn((double)t.out[r], (double)total);
    cdf = __dadd_rn(cdf, d);
    t.dist[r] = d;
    t.cdf[r] = cdf;
  }
}

// the first i in [0, n) with a[i] >= u (a nondecreasing), n if none: the reference's linear scan
__device__ __forceinline__ int first_at_least(const double* __restrict__ a, int n, double u) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] >= u) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

// u of walk w, step t: the top 53 bits of splitmix(splitmix(root, w), t) over 2^53, root = splitmix(~seed, 0)
__device__ __forceinline__ double walk_uniform(uint64_t root, int w, int t) {
  return (double)(splitmix(splitmix(root, (uint64_t)w), (uint64_t)t) >> 11) * 0x1p-53;
}

__global__ void ge_walk_kernel(Transitions t, uint64_t root, int W, int L, int32_t* __restrict__ walks,
                               int32_t* __restrict__ lengths) {
  const int S = t.n_rows[0];
  for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < W; w += gridDim.x * blockDim.x) {
    int32_t* out = walks + (int64_t)w * L;
    int len = 0;
    const int r0 = first_at_least(t.cdf, S, walk_uniform(root, w, 0));
    if (r0 < S) {                                        // past the last cumulative sum: an empty walk
      int cur = t.source[r0];
      out[len++] = cur;
      for (int step = 1; step < L; ++step) {
        const int r = t.row_of[cur];
        if (r < 0) break;                                // no outgoing pair: the walk ends
        const int lo = t.row_ptr[r], hi = t.row_ptr[r + 1];
        const int e = lo + first_at_least(t.cum + lo, hi - lo, walk_uniform(root, w, step));
        if (e < hi) cur = t.target[e];                   // past the row's last sum: the current item repeats
        out[len++] = cur;
      }
    }
    lengths[w] = len;
    for (int i = len; i < L; ++i) out[i] = -1;
  }
}

// the walks as a corpus: word i = walks[i] for the steps inside its walk, keyed by the walk
__global__ void ge_flat_kernel(const int32_t* __restrict__ lengths, int64_t n, int L, uint8_t* __restrict__ flag,
                               uint32_t* __restrict__ key) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int w = (int)(i / L);
    flag[i] = (int)(i - (int64_t)w * L) < lengths[w];
    key[i] = (uint32_t)w;
  }
}

int build_transitions(Scratch& sc, cudaStream_t s, const I2vCorpus& c, int n, int32_t n_slots, Transitions* t) {
  uint64_t *d_key, *d_skey, *d_ukey;
  int32_t *d_iota, *d_runs, *d_rstart;
  uint8_t* d_flag;
  int* d_nruns;
  GE_TRY(sc.alloc(&d_key, n)); GE_TRY(sc.alloc(&d_skey, n)); GE_TRY(sc.alloc(&d_ukey, n));
  GE_TRY(sc.alloc(&d_iota, n)); GE_TRY(sc.alloc(&d_runs, n)); GE_TRY(sc.alloc(&d_rstart, n));
  GE_TRY(sc.alloc(&d_flag, n)); GE_TRY(sc.alloc(&d_nruns, 1));
  GE_TRY(sc.alloc(&t->source, n)); GE_TRY(sc.alloc(&t->row_ptr, n + 1)); GE_TRY(sc.alloc(&t->out, n));
  GE_TRY(sc.alloc(&t->dist, n)); GE_TRY(sc.alloc(&t->cdf, n)); GE_TRY(sc.alloc(&t->target, n));
  GE_TRY(sc.alloc(&t->count, n)); GE_TRY(sc.alloc(&t->prob, n)); GE_TRY(sc.alloc(&t->cum, n));
  GE_TRY(sc.alloc(&t->row_of, n_slots)); GE_TRY(sc.alloc(&t->n_rows, 2));
  GE_TRY(cudaMemsetAsync(t->row_of, 0xff, sizeof(int32_t) * n_slots, s));
  const int T = 256;
  ge_pair_kernel<<<grid_for(n, T), T, 0, s>>>(c.movie, c.user, c.n, n, d_key, d_iota);
  GE_LAUNCHED();
  size_t b1 = 0, b2 = 0, b3 = 0;
  GE_TRY(cub::DeviceRadixSort::SortKeys(nullptr, b1, d_key, d_skey, n, 0, 49, s));
  GE_TRY(cub::DeviceRunLengthEncode::Encode(nullptr, b2, d_skey, d_ukey, d_runs, d_nruns, n, s));
  GE_TRY(cub::DeviceSelect::Flagged(nullptr, b3, d_iota, d_flag, d_rstart, t->n_rows, n, s));
  const size_t tmp_bytes = std::max(b1, std::max(b2, b3));
  uint8_t* d_tmp;
  GE_TRY(sc.alloc(&d_tmp, tmp_bytes));
  GE_TRY(cub::DeviceRadixSort::SortKeys(d_tmp, b1, d_key, d_skey, n, 0, 49, s));
  GE_TRY(cub::DeviceRunLengthEncode::Encode(d_tmp, b2, d_skey, d_ukey, d_runs, d_nruns, n, s));
  ge_row_flag_kernel<<<grid_for(n, T), T, 0, s>>>(d_ukey, d_nruns, n, d_flag);
  GE_LAUNCHED();
  GE_TRY(cub::DeviceSelect::Flagged(d_tmp, b3, d_iota, d_flag, d_rstart, t->n_rows, n, s));
  ge_row_kernel<<<grid_for(n, T), T, 0, s>>>(d_ukey, d_runs, d_nruns, d_rstart, *t);
  GE_LAUNCHED();
  ge_dist_kernel<<<1, 32, 0, s>>>(d_ukey, d_nruns, *t);
  GE_LAUNCHED();
  return SRS_OK;
}

// the ratings' checks, the device, the sentences and the transitions
struct GraphCall {
  Scratch sc;
  StreamGuard sg;
  I2vCorpus corpus;
  Transitions t;
  int32_t n_slots = 0;
  int n = 0;
};

int begin(GraphCall& g, const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
          const int32_t* timestamp, int64_t n_ratings, int32_t device) {
  if (int rc = i2v_select_device(device)) return rc;
  GE_TRY(cudaStreamCreateWithFlags(&g.sg.s, cudaStreamNonBlocking));
  g.n = (int)n_ratings;
  if (int rc = i2v_positive_corpus(g.sc, g.sg.s, user_id, movie_id, half, timestamp, g.n, &g.corpus)) return rc;
  return build_transitions(g.sc, g.sg.s, g.corpus, g.n, g.n_slots, &g.t);
}

int check_walks(int32_t num_walks, int32_t walk_length) {
  if (num_walks < 1 || walk_length < 1 || (int64_t)num_walks * walk_length > kMaxWalkWords)
    return ge_fail(SRS_ERR_INVALID, "%d walks of length %d: both must be >= 1 and their product <= %lld", num_walks,
                   walk_length, (long long)kMaxWalkWords);
  return SRS_OK;
}

int run_walks(GraphCall& g, int32_t num_walks, int32_t walk_length, uint64_t seed, int32_t** d_walks,
              int32_t** d_len) {
  const int64_t nw = (int64_t)num_walks * walk_length;
  GE_TRY(g.sc.alloc(d_walks, nw));
  GE_TRY(g.sc.alloc(d_len, num_walks));
  const int T = 128;
  ge_walk_kernel<<<grid_for(num_walks, T), T, 0, g.sg.s>>>(g.t, splitmix(~seed, 0), num_walks, walk_length,
                                                           *d_walks, *d_len);
  GE_LAUNCHED();
  return SRS_OK;
}

}  // namespace
}  // namespace srs

using namespace srs;

extern "C" int srs_item_transitions_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                                         const int32_t* timestamp, int64_t n_ratings, int32_t device,
                                         int32_t source_capacity, int32_t edge_capacity, int32_t* sources,
                                         int32_t* row_offsets, int32_t* out_counts, double* source_probs,
                                         int32_t* targets, int32_t* counts, double* probs, int32_t* n_sources,
                                         int32_t* n_edges) {
  if (!n_sources || !n_edges) return ge_fail(SRS_ERR_INVALID, "null n_sources or n_edges");
  *n_sources = *n_edges = 0;
  if (source_capacity < 0 || edge_capacity < 0 ||
      (source_capacity > 0 && (!sources || !row_offsets || !out_counts || !source_probs)) ||
      (edge_capacity > 0 && (!targets || !counts || !probs)))
    return ge_fail(SRS_ERR_INVALID, "negative capacity or null outputs");
  GraphCall g;
  if (int rc = i2v_check_ratings(user_id, movie_id, half, timestamp, n_ratings, &g.n_slots)) return rc;
  if (int rc = begin(g, user_id, movie_id, half, timestamp, n_ratings, device)) return rc;
  cudaStream_t s = g.sg.s;
  int se[2];
  GE_TRY(cudaMemcpyAsync(se, g.t.n_rows, sizeof(se), cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaStreamSynchronize(s));
  if (se[0] > source_capacity || se[1] > edge_capacity)
    return ge_fail(SRS_ERR_RANGE, "%d sources and %d pairs exceed the capacities %d and %d", se[0], se[1],
                   source_capacity, edge_capacity);
  GE_TRY(cudaMemcpyAsync(sources, g.t.source, sizeof(int32_t) * se[0], cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaMemcpyAsync(row_offsets, g.t.row_ptr, sizeof(int32_t) * (se[0] + 1), cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaMemcpyAsync(out_counts, g.t.out, sizeof(int32_t) * se[0], cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaMemcpyAsync(source_probs, g.t.dist, sizeof(double) * se[0], cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaMemcpyAsync(targets, g.t.target, sizeof(int32_t) * se[1], cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaMemcpyAsync(counts, g.t.count, sizeof(int32_t) * se[1], cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaMemcpyAsync(probs, g.t.prob, sizeof(double) * se[1], cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaStreamSynchronize(s));
  *n_sources = se[0];
  *n_edges = se[1];
  return SRS_OK;
}

extern "C" int srs_random_walks_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                                     const int32_t* timestamp, int64_t n_ratings, int32_t num_walks,
                                     int32_t walk_length, uint64_t seed, int32_t device, int32_t* walks,
                                     int32_t* lengths) {
  if (int rc = check_walks(num_walks, walk_length)) return rc;
  if (!walks || !lengths) return ge_fail(SRS_ERR_INVALID, "null outputs");
  GraphCall g;
  if (int rc = i2v_check_ratings(user_id, movie_id, half, timestamp, n_ratings, &g.n_slots)) return rc;
  if (int rc = begin(g, user_id, movie_id, half, timestamp, n_ratings, device)) return rc;
  int32_t *d_walks, *d_len;
  if (int rc = run_walks(g, num_walks, walk_length, seed, &d_walks, &d_len)) return rc;
  cudaStream_t s = g.sg.s;
  GE_TRY(cudaMemcpyAsync(walks, d_walks, sizeof(int32_t) * num_walks * (int64_t)walk_length, cudaMemcpyDeviceToHost,
                         s));
  GE_TRY(cudaMemcpyAsync(lengths, d_len, sizeof(int32_t) * num_walks, cudaMemcpyDeviceToHost, s));
  GE_TRY(cudaStreamSynchronize(s));
  return SRS_OK;
}

extern "C" int srs_graph_embedding_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                                        const int32_t* timestamp, int64_t n_ratings,
                                        const srs_item2vec_params* params, int32_t num_walks, int32_t walk_length,
                                        int32_t device, int32_t capacity, int32_t* vocab_ids, float* vectors,
                                        int32_t* vocab_size) {
  if (!vocab_size) return ge_fail(SRS_ERR_INVALID, "null vocab_size");
  *vocab_size = 0;
  if (int rc = i2v_check_params(params)) return rc;
  if (int rc = check_walks(num_walks, walk_length)) return rc;
  if (capacity < 0 || (capacity > 0 && (!vocab_ids || !vectors)))
    return ge_fail(SRS_ERR_INVALID, "negative capacity or null outputs");
  GraphCall g;
  if (int rc = i2v_check_ratings(user_id, movie_id, half, timestamp, n_ratings, &g.n_slots)) return rc;
  if (int rc = begin(g, user_id, movie_id, half, timestamp, n_ratings, device)) return rc;
  int32_t *d_walks, *d_len;
  if (int rc = run_walks(g, num_walks, walk_length, params->seed, &d_walks, &d_len)) return rc;
  cudaStream_t s = g.sg.s;
  const int64_t nw = (int64_t)num_walks * walk_length;
  uint8_t *d_flag, *d_tmp;
  uint32_t *d_key, *d_wkey;
  int32_t* d_words;
  int* d_n;
  GE_TRY(g.sc.alloc(&d_flag, nw)); GE_TRY(g.sc.alloc(&d_key, nw)); GE_TRY(g.sc.alloc(&d_wkey, nw));
  GE_TRY(g.sc.alloc(&d_words, nw)); GE_TRY(g.sc.alloc(&d_n, 1));
  const int T = 256;
  ge_flat_kernel<<<grid_for(nw, T), T, 0, s>>>(d_len, nw, walk_length, d_flag, d_key);
  GE_LAUNCHED();
  size_t tmp_bytes = 0;
  GE_TRY(cub::DeviceSelect::Flagged(nullptr, tmp_bytes, d_walks, d_flag, d_words, d_n, (int)nw, s));
  GE_TRY(g.sc.alloc(&d_tmp, tmp_bytes));
  GE_TRY(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_walks, d_flag, d_words, d_n, (int)nw, s));
  GE_TRY(cub::DeviceSelect::Flagged(d_tmp, tmp_bytes, d_key, d_flag, d_wkey, d_n, (int)nw, s));
  return word2vec_fit(g.sc, s, d_words, d_wkey, d_n, (int)nw, g.n_slots, *params, "occurrences in the walks",
                      capacity, vocab_ids, vectors, vocab_size);
}
