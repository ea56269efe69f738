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

#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"

namespace srs {
namespace {

constexpr int64_t kMaxWalkWords = 21000000;   // num_walks * walk_length: item2vec's bound on the corpus
constexpr uint64_t kSentinel = 1ull << 48;
constexpr uint32_t kIdMask = (1u << 24) - 1;

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

// u of walk w, step t, root = splitmix(~seed, 0)
__device__ __forceinline__ double walk_uniform(uint64_t root, int w, int t) {
  return uniform53(splitmix(root, (uint64_t)w), (uint64_t)t);
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

int build_transitions(HostCall& hc, const I2vCorpus& c, int n, int32_t n_slots, Transitions* t) {
  Scratch& sc = hc.sc;
  cudaStream_t s = hc.s;
  uint64_t *d_key, *d_skey, *d_ukey;
  int32_t *d_iota, *d_runs, *d_rstart;
  uint8_t* d_flag;
  int* d_nruns;
  CUDA_TRY(sc.alloc(&d_key, n)); CUDA_TRY(sc.alloc(&d_skey, n)); CUDA_TRY(sc.alloc(&d_ukey, n));
  CUDA_TRY(sc.alloc(&d_iota, n)); CUDA_TRY(sc.alloc(&d_runs, n)); CUDA_TRY(sc.alloc(&d_rstart, n));
  CUDA_TRY(sc.alloc(&d_flag, n)); CUDA_TRY(sc.alloc(&d_nruns, 1));
  CUDA_TRY(sc.alloc(&t->source, n)); CUDA_TRY(sc.alloc(&t->row_ptr, n + 1)); CUDA_TRY(sc.alloc(&t->out, n));
  CUDA_TRY(sc.alloc(&t->dist, n)); CUDA_TRY(sc.alloc(&t->cdf, n)); CUDA_TRY(sc.alloc(&t->target, n));
  CUDA_TRY(sc.alloc(&t->count, n)); CUDA_TRY(sc.alloc(&t->prob, n)); CUDA_TRY(sc.alloc(&t->cum, n));
  CUDA_TRY(sc.alloc(&t->row_of, n_slots)); CUDA_TRY(sc.alloc(&t->n_rows, 2));
  CUDA_TRY(cudaMemsetAsync(t->row_of, 0xff, sizeof(int32_t) * n_slots, s));
  const int T = 256;
  ge_pair_kernel<<<grid_for(n, T), T, 0, s>>>(c.movie, c.user, c.n, n, d_key, d_iota);
  LAUNCHED();
  CUB_RUN(hc, cub::DeviceRadixSort::SortKeys(tmp__, tb__, d_key, d_skey, n, 0, 49, s));
  CUB_RUN(hc, cub::DeviceRunLengthEncode::Encode(tmp__, tb__, d_skey, d_ukey, d_runs, d_nruns, n, s));
  ge_row_flag_kernel<<<grid_for(n, T), T, 0, s>>>(d_ukey, d_nruns, n, d_flag);
  LAUNCHED();
  CUB_RUN(hc, cub::DeviceSelect::Flagged(tmp__, tb__, d_iota, d_flag, d_rstart, t->n_rows, n, s));
  ge_row_kernel<<<grid_for(n, T), T, 0, s>>>(d_ukey, d_runs, d_nruns, d_rstart, *t);
  LAUNCHED();
  ge_dist_kernel<<<1, 32, 0, s>>>(d_ukey, d_nruns, *t);
  LAUNCHED();
  return SRS_OK;
}

// a host call with the sentences and the transitions of its ratings
struct GraphCall : HostCall {
  I2vCorpus corpus;
  Transitions t;
  int32_t n_slots = 0;
  int n = 0;
};

int begin_graph(GraphCall& g, const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                const int32_t* timestamp, int64_t n_ratings, int32_t device) {
  PROPAGATE(g.begin(device));
  g.n = (int)n_ratings;
  PROPAGATE(i2v_positive_corpus(g, user_id, movie_id, half, timestamp, g.n, &g.corpus));
  return build_transitions(g, g.corpus, g.n, g.n_slots, &g.t);
}

int check_walks(int32_t num_walks, int32_t walk_length) {
  if (num_walks < 1 || walk_length < 1 || (int64_t)num_walks * walk_length > kMaxWalkWords)
    return failf(SRS_ERR_INVALID, "%d walks of length %d: both must be >= 1 and their product <= %lld", num_walks,
                   walk_length, (long long)kMaxWalkWords);
  return SRS_OK;
}

int run_walks(GraphCall& g, int32_t num_walks, int32_t walk_length, uint64_t seed, int32_t** d_walks,
              int32_t** d_len) {
  const int64_t nw = (int64_t)num_walks * walk_length;
  CUDA_TRY(g.sc.alloc(d_walks, nw));
  CUDA_TRY(g.sc.alloc(d_len, num_walks));
  const int T = 128;
  ge_walk_kernel<<<grid_for(num_walks, T), T, 0, g.s>>>(g.t, splitmix(~seed, 0), num_walks, walk_length,
                                                           *d_walks, *d_len);
  LAUNCHED();
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
  if (!n_sources || !n_edges) return failf(SRS_ERR_INVALID, "null n_sources or n_edges");
  *n_sources = *n_edges = 0;
  if (source_capacity < 0 || edge_capacity < 0 ||
      (source_capacity > 0 && (!sources || !row_offsets || !out_counts || !source_probs)) ||
      (edge_capacity > 0 && (!targets || !counts || !probs)))
    return failf(SRS_ERR_INVALID, "negative capacity or null outputs");
  GraphCall g;
  PROPAGATE(i2v_check_ratings(user_id, movie_id, half, timestamp, n_ratings, &g.n_slots));
  PROPAGATE(begin_graph(g, user_id, movie_id, half, timestamp, n_ratings, device));
  cudaStream_t s = g.s;
  int se[2];
  CUDA_TRY(cudaMemcpyAsync(se, g.t.n_rows, sizeof(se), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  if (se[0] > source_capacity || se[1] > edge_capacity)
    return failf(SRS_ERR_RANGE, "%d sources and %d pairs exceed the capacities %d and %d", se[0], se[1],
                   source_capacity, edge_capacity);
  CUDA_TRY(cudaMemcpyAsync(sources, g.t.source, sizeof(int32_t) * se[0], cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(row_offsets, g.t.row_ptr, sizeof(int32_t) * (se[0] + 1), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out_counts, g.t.out, sizeof(int32_t) * se[0], cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(source_probs, g.t.dist, sizeof(double) * se[0], cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(targets, g.t.target, sizeof(int32_t) * se[1], cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(counts, g.t.count, sizeof(int32_t) * se[1], cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(probs, g.t.prob, sizeof(double) * se[1], cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  *n_sources = se[0];
  *n_edges = se[1];
  return SRS_OK;
}

extern "C" int srs_random_walks_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                                     const int32_t* timestamp, int64_t n_ratings, int32_t num_walks,
                                     int32_t walk_length, uint64_t seed, int32_t device, int32_t* walks,
                                     int32_t* lengths) {
  PROPAGATE(check_walks(num_walks, walk_length));
  if (!walks || !lengths) return failf(SRS_ERR_INVALID, "null outputs");
  GraphCall g;
  PROPAGATE(i2v_check_ratings(user_id, movie_id, half, timestamp, n_ratings, &g.n_slots));
  PROPAGATE(begin_graph(g, user_id, movie_id, half, timestamp, n_ratings, device));
  int32_t *d_walks, *d_len;
  PROPAGATE(run_walks(g, num_walks, walk_length, seed, &d_walks, &d_len));
  cudaStream_t s = g.s;
  CUDA_TRY(cudaMemcpyAsync(walks, d_walks, sizeof(int32_t) * num_walks * (int64_t)walk_length, cudaMemcpyDeviceToHost,
                         s));
  CUDA_TRY(cudaMemcpyAsync(lengths, d_len, sizeof(int32_t) * num_walks, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  return SRS_OK;
}

extern "C" int srs_graph_embedding_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                                        const int32_t* timestamp, int64_t n_ratings,
                                        const srs_item2vec_params* params, int32_t num_walks, int32_t walk_length,
                                        int32_t device, int32_t capacity, int32_t* vocab_ids, float* vectors,
                                        int32_t* vocab_size) {
  if (!vocab_size) return failf(SRS_ERR_INVALID, "null vocab_size");
  *vocab_size = 0;
  PROPAGATE(i2v_check_params(params));
  PROPAGATE(check_walks(num_walks, walk_length));
  if (capacity < 0 || (capacity > 0 && (!vocab_ids || !vectors)))
    return failf(SRS_ERR_INVALID, "negative capacity or null outputs");
  GraphCall g;
  PROPAGATE(i2v_check_ratings(user_id, movie_id, half, timestamp, n_ratings, &g.n_slots));
  PROPAGATE(begin_graph(g, user_id, movie_id, half, timestamp, n_ratings, device));
  int32_t *d_walks, *d_len;
  PROPAGATE(run_walks(g, num_walks, walk_length, params->seed, &d_walks, &d_len));
  cudaStream_t s = g.s;
  const int64_t nw = (int64_t)num_walks * walk_length;
  uint8_t* d_flag;
  uint32_t *d_key, *d_wkey;
  int32_t* d_words;
  int* d_n;
  CUDA_TRY(g.sc.alloc(&d_flag, nw)); CUDA_TRY(g.sc.alloc(&d_key, nw)); CUDA_TRY(g.sc.alloc(&d_wkey, nw));
  CUDA_TRY(g.sc.alloc(&d_words, nw)); CUDA_TRY(g.sc.alloc(&d_n, 1));
  const int T = 256;
  ge_flat_kernel<<<grid_for(nw, T), T, 0, s>>>(d_len, nw, walk_length, d_flag, d_key);
  LAUNCHED();
  CUB_RUN(g, cub::DeviceSelect::Flagged(tmp__, tb__, d_walks, d_flag, d_words, d_n, (int)nw, s));
  CUB_RUN(g, cub::DeviceSelect::Flagged(tmp__, tb__, d_key, d_flag, d_wkey, d_n, (int)nw, s));
  return word2vec_fit(g, d_words, d_wkey, d_n, (int)nw, g.n_slots, *params, "occurrences in the walks",
                      capacity, vocab_ids, vectors, vocab_size);
}
