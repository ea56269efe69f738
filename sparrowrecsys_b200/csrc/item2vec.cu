// item2vec.cu - the reference's Embedding job (Embedding.scala:27-138) on one device: Spark MLlib's Word2Vec
// (hierarchical-softmax skip-gram, SGD) over each user's positive ratings, and the user embeddings.  DESIGN.md
// section 4.12 gives the semantics, the orders Spark leaves open and the bounds.
//
// srs_item2vec_host, on one stream.  i2v_positive_corpus (steps 1-2) builds the sentences; word2vec_fit (steps 3-7)
// is Word2Vec.fit over any device corpus given as movie ids plus sentence keys, and graphemb.cu trains it on random
// walks as well:
//   1. user_time_order (featureeng.cu)   (user, timestamp string, file index) order of the ratings;
//   2. i2v_flag_kernel + DeviceSelect    the positive ratings (>= 3.5) in that order, and i2v_gather_kernel their
//                                        movies and users: the words and their sentence keys;
//   3. i2v_count_kernel                  a per-movie count (integer atomics);
//   -- the counts come to the host: vocabulary (count >= 5, count descending, id ascending) and Huffman tree --
//   4. i2v_map_kernel + two selects      the in-vocabulary words and their users;
//   5. i2v_user_start_kernel, a max-scan, i2v_chunk_kernel + select: sentence starts, cut every 1000 words;
//   6. i2v_init_kernel                   syn0 from the counter-based generator, syn1 = 0;
//   7. per iteration (no host round trip): [i2v_broadcast_kernel] i2v_train_kernel [i2v_merge_kernel] - the
//      bracketed launches only with more than one partition, whose copies of the tables then live in global memory.
// i2v_train_kernel runs one warp per partition.  Per (centre word, context word) pair the lanes first take the
// centre word's Huffman path nodes (at most 32): each lane's dot product and g; then the lanes take the dimensions
// (at most 64, two per lane): neu1e summed over the nodes in path order and the syn1 / syn0 updates.  The dots of
// one path are independent (its nodes are distinct rows of syn1 and syn0 changes only after the path), so this is
// the sequential loop's arithmetic exactly.  Every float operation is an explicitly rounded intrinsic: no
// multiply-add is fused, so the results equal oracle/item2vec_c.c bit for bit.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"

namespace srs {
namespace {

constexpr int kMinCount = 5;           // Spark's defaults
constexpr int kMaxSentence = 1000;
constexpr double kLearningRate = 0.025;
constexpr int kExpTable = 1000;
constexpr int kMaxExp = 6;
constexpr int kMaxCode = 32;           // one lane per path node
constexpr int kMaxDim = 64;            // two dimensions per lane
constexpr int64_t kMaxRatings = 21000000;
constexpr int32_t kMaxMovieSlots = 1 << 24;
constexpr int kMaxWindow = 1 << 16;
constexpr int kMaxIterations = 100000;
constexpr int kMaxPartitions = 1 << 16;
constexpr unsigned kFull = 0xffffffffu;

struct MaxOp {
  __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};

__global__ void i2v_flag_kernel(const int32_t* __restrict__ order, const int8_t* __restrict__ half, int n,
                                uint8_t* __restrict__ flag, int32_t* __restrict__ iota) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    flag[i] = half[order[i]] >= 7;                      // rating >= 3.5
    iota[i] = i;
  }
}

__global__ void i2v_gather_kernel(const int32_t* __restrict__ sel, const int* __restrict__ n_sel,
                                  const int32_t* __restrict__ order, const uint32_t* __restrict__ suser,
                                  const int32_t* __restrict__ movie, int32_t* __restrict__ pmovie,
                                  uint32_t* __restrict__ puser) {
  const int n = *n_sel;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int s = sel[i];
    pmovie[i] = movie[order[s]];
    puser[i] = suser[s];
  }
}

__global__ void i2v_count_kernel(const int32_t* __restrict__ words, const int* __restrict__ n_words,
                                 int32_t* __restrict__ count) {
  const int n = *n_words;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) atomicAdd(count + words[i], 1);
}

// flags every one of the n entries: those past the positives are cleared for the selects that follow
__global__ void i2v_map_kernel(const int32_t* __restrict__ pmovie, const int* __restrict__ n_pos, int n,
                               const int32_t* __restrict__ vocab_index, int32_t* __restrict__ pword,
                               uint8_t* __restrict__ flag) {
  const int np = *n_pos;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int w = i < np ? vocab_index[pmovie[i]] : -1;
    pword[i] = w;
    flag[i] = w >= 0;
  }
}

__global__ void i2v_user_start_kernel(const uint32_t* __restrict__ wuser, int n, int32_t* __restrict__ start) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    start[i] = (i == 0 || wuser[i] != wuser[i - 1]) ? i : 0;
}

// after the max-scan, ustart[i] = first word of word i's user: a sentence starts every 1000 words of a user
__global__ void i2v_chunk_kernel(const int32_t* __restrict__ ustart, int n, uint8_t* __restrict__ flag,
                                 int32_t* __restrict__ iota) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    flag[i] = (i - ustart[i]) % kMaxSentence == 0;
    iota[i] = i;
  }
}

// syn0 = (u - 0.5f) / vectorSize, u from the top 24 bits of splitmix(seed, element)
__global__ void i2v_init_kernel(float* __restrict__ syn0, int64_t n, uint64_t seed, int D) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float u = __fmul_rn((float)(uint32_t)(splitmix(seed, (uint64_t)i) >> 40), 1.0f / 16777216.0f);
    syn0[i] = __fdiv_rn(__fsub_rn(u, 0.5f), (float)D);
  }
}

__global__ void i2v_broadcast_kernel(const float* __restrict__ glob, int64_t vd, int P, float* __restrict__ local) {
  const int64_t n = vd * P;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    local[i] = glob[i % vd];
}

// a row modified by one or more partitions = their rows summed in partition order, times 1.0f / count
__global__ void i2v_merge_kernel(const float* __restrict__ local, const uint8_t* __restrict__ mod, int V, int D,
                                 int P, float* __restrict__ glob) {
  const int64_t vd = (int64_t)V * D;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < vd; e += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / D);
    int cnt = 0;
    float v = 0.f;
    for (int p = 0; p < P; ++p) {
      if (!mod[(int64_t)p * V + r]) continue;
      const float x = local[(int64_t)p * vd + e];
      v = cnt++ ? __fadd_rn(v, x) : x;
    }
    if (cnt) glob[e] = __fmul_rn(v, __fdiv_rn(1.0f, (float)cnt));
  }
}

struct TrainArgs {
  const int32_t* words;                // [n_words] vocabulary indices, sentence after sentence
  const int32_t* chunk_offs;           // [*n_chunks] first word of each sentence
  const int* n_chunks;
  int n_words;
  const uint32_t* code_bits;           // [V] bit d = code of path node d
  const int32_t* points;               // [V][32] path nodes (rows of syn1)
  const int32_t* codelen;              // [V]
  const float* exp_table;              // [1000]
  float* syn0;                         // [P][V][D]
  float* syn1;                         // [P][V][D]
  uint8_t* mod0;                       // [P][V], nullptr with one partition
  uint8_t* mod1;
  int V, D, window, iterations, P;
  uint64_t seed;
  int64_t train_words;
  double lr;
};

// One warp per partition: the partition's sentences in order, one (centre word, context word) pair at a time.
__global__ void __launch_bounds__(128) i2v_train_kernel(TrainArgs a, int k) {
  const int p = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= a.P) return;
  const int D = a.D, V = a.V, window = a.window;
  const int64_t vd = (int64_t)V * D;
  float* s0 = a.syn0 + p * vd;
  float* s1 = a.syn1 + p * vd;
  const uint64_t kp = splitmix(splitmix(~a.seed, (uint64_t)k), (uint64_t)p);
  const int n_chunks = *a.n_chunks;
  double alpha = a.lr;
  int64_t wc = 0, lwc = 0;
  for (int i = p; i < n_chunks; i += a.P) {
    if (wc - lwc > 10000) {
      lwc = wc;
      const double num = __dadd_rn(__dmul_rn((double)a.P, (double)wc), (double)((int64_t)(k - 1) * a.train_words));
      const double frac = __ddiv_rn(num, (double)((int64_t)a.iterations * a.train_words + 1));
      alpha = __dmul_rn(a.lr, __dsub_rn(1.0, frac));
      const double floor_ = __dmul_rn(a.lr, 0.0001);
      if (alpha < floor_) alpha = floor_;
    }
    const int lo = a.chunk_offs[i];
    const int n = (i + 1 < n_chunks ? a.chunk_offs[i + 1] : a.n_words) - lo;
    wc += n;
    const int32_t* sent = a.words + lo;
    for (int pos = 0; pos < n; ++pos) {
      const int word = sent[pos];
      const int b = (int)((splitmix(kp, (uint64_t)(lo + pos)) >> 32) % (uint64_t)window);
      const int L = a.codelen[word];
      const bool node = lane < L;
      const int my_pt = node ? a.points[(int64_t)word * kMaxCode + lane] : 0;
      const float my_c = (float)(1 - (int)((a.code_bits[word] >> lane) & 1u));     // (float)(1 - code)
      const float* r1 = s1 + (int64_t)my_pt * D;
      for (int aa = b; aa < 2 * window + 1 - b; ++aa) {
        if (aa == window) continue;
        const int c = pos - window + aa;
        if (c < 0 || c >= n) continue;
        const int last = sent[c];
        float* r0 = s0 + (int64_t)last * D;
        const float x0a = lane < D ? r0[lane] : 0.f;
        const float x0b = lane + 32 < D ? r0[lane + 32] : 0.f;
        float f = 0.f;                                   // sdot, sequential over the dimensions
        for (int j = 0; j < D; ++j) {
          const float xj = __shfl_sync(kFull, j < 32 ? x0a : x0b, j & 31);
          if (node) f = __fadd_rn(f, __fmul_rn(xj, r1[j]));
        }
        const bool ok = node && f > -(float)kMaxExp && f < (float)kMaxExp;
        float g = 0.f;
        if (ok) {
          const int ind = (int)__dmul_rn((double)__fadd_rn(f, (float)kMaxExp), 83.0);   // 1000 / 6 / 2.0
          g = (float)__dmul_rn((double)__fsub_rn(my_c, a.exp_table[ind]), alpha);
          if (a.mod1) a.mod1[(int64_t)p * V + my_pt] = 1;
        }
        const unsigned okm = __ballot_sync(kFull, ok);   // also orders every lane's dot before the updates
        float na = 0.f, nb = 0.f;
        for (unsigned m = okm; m; m &= m - 1) {          // the path's nodes in order
          const int d = __ffs(m) - 1;
          const float gd = __shfl_sync(kFull, g, d);
          float* q = s1 + (int64_t)__shfl_sync(kFull, my_pt, d) * D;
          if (lane < D) {
            const float sv = q[lane];
            na = __fadd_rn(na, __fmul_rn(gd, sv));       // neu1e += g syn1 (before its update)
            q[lane] = __fadd_rn(sv, __fmul_rn(gd, x0a)); // syn1 += g syn0
          }
          if (lane + 32 < D) {
            const float sv = q[lane + 32];
            nb = __fadd_rn(nb, __fmul_rn(gd, sv));
            q[lane + 32] = __fadd_rn(sv, __fmul_rn(gd, x0b));
          }
        }
        if (lane < D) r0[lane] = __fadd_rn(x0a, na);
        if (lane + 32 < D) r0[lane + 32] = __fadd_rn(x0b, nb);
        if (lane == 0 && a.mod0) a.mod0[(int64_t)p * V + last] = 1;
        __syncwarp();                                    // the next pair's dots read what the lanes wrote
      }
    }
  }
}

// One warp per user: the user's ratings from last to first in file order, lanes over the dimensions.
__global__ void i2v_user_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ start,
                                const int32_t* __restrict__ count, const int* __restrict__ n_users,
                                const int32_t* __restrict__ movie, const int32_t* __restrict__ row_of,
                                const float* __restrict__ vec, int D, float* __restrict__ out) {
  const int u = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (u >= *n_users) return;
  float acc_a = 0.f, acc_b = 0.f;
  const int s = start[u];
  for (int r = s + count[u] - 1; r >= s; --r) {
    const int row = row_of[movie[order[r]]];
    if (row < 0) continue;
    const float* v = vec + (int64_t)row * D;
    if (lane < D) acc_a = __fadd_rn(acc_a, v[lane]);
    if (lane + 32 < D) acc_b = __fadd_rn(acc_b, v[lane + 32]);
  }
  if (lane < D) out[(int64_t)u * D + lane] = acc_a;
  if (lane + 32 < D) out[(int64_t)u * D + lane + 32] = acc_b;
}

// createBinaryTree (word2vec.c's, as Spark restates it): codes and points of each word, root first.  Returns
// the longest code length.
int huffman(const std::vector<int64_t>& cn, std::vector<uint32_t>& code_bits, std::vector<int32_t>& points,
            std::vector<int32_t>& codelen) {
  const int V = (int)cn.size();
  std::vector<int64_t> count(2 * V + 1, 0);
  std::vector<int32_t> binary(2 * V + 1, 0), parent(2 * V + 1, 0);
  for (int a = 0; a < V; ++a) count[a] = cn[a];
  for (int a = V; a < 2 * V; ++a) count[a] = 1000000000;
  int pos1 = V - 1, pos2 = V;
  for (int a = 0; a < V - 1; ++a) {
    int mins[2];
    for (int t = 0; t < 2; ++t) {
      if (pos1 >= 0 && count[pos1] < count[pos2]) mins[t] = pos1--;
      else mins[t] = pos2++;
    }
    count[V + a] = count[mins[0]] + count[mins[1]];
    parent[mins[0]] = parent[mins[1]] = V + a;
    binary[mins[1]] = 1;
  }
  code_bits.assign(V, 0);
  points.assign((size_t)V * kMaxCode, 0);
  codelen.assign(V, 0);
  int deepest = 0;
  std::vector<int32_t> cs, ps;
  for (int a = 0; a < V; ++a) {
    cs.clear();
    ps.clear();
    for (int b = a; b != 2 * V - 2; b = parent[b]) {
      cs.push_back(binary[b]);
      ps.push_back(b);
    }
    const int len = (int)cs.size();
    deepest = std::max(deepest, len);
    if (len > kMaxCode) continue;
    codelen[a] = len;
    for (int b = 0; b < len; ++b) {
      if (cs[b]) code_bits[a] |= 1u << (len - b - 1);
      if (len - b < len) points[(size_t)a * kMaxCode + (len - b)] = ps[b] - V;
    }
    if (len > 0) points[(size_t)a * kMaxCode] = V - 2;
  }
  return deepest;
}

int check_ratings(const int32_t* user_id, const int32_t* movie_id, int64_t n_ratings, int32_t* n_slots) {
  if (n_ratings < 0 || n_ratings > kMaxRatings)
    return failf(SRS_ERR_INVALID, "n_ratings %lld outside 0..%lld", (long long)n_ratings, (long long)kMaxRatings);
  if (n_ratings && (!user_id || !movie_id)) return failf(SRS_ERR_INVALID, "null ratings");
  int32_t mx = -1;
  for (int64_t i = 0; i < n_ratings; ++i) {
    if (user_id[i] < 0 || movie_id[i] < 0)
      return failf(SRS_ERR_INVALID, "rating %lld: negative id (user %d, movie %d)", (long long)i, user_id[i],
                      movie_id[i]);
    if (movie_id[i] >= kMaxMovieSlots)
      return failf(SRS_ERR_INVALID, "rating %lld: movie id %d is not below 2^24", (long long)i, movie_id[i]);
    mx = std::max(mx, movie_id[i]);
  }
  *n_slots = mx + 1;
  return SRS_OK;
}

}  // namespace

int i2v_check_params(const srs_item2vec_params* params) {
  if (!params) return failf(SRS_ERR_INVALID, "null params");
  const srs_item2vec_params& hp = *params;
  if (hp.vector_size < 1 || hp.vector_size > kMaxDim)
    return failf(SRS_ERR_INVALID, "vector_size %d outside 1..%d", hp.vector_size, kMaxDim);
  if (hp.window < 1 || hp.window > kMaxWindow)
    return failf(SRS_ERR_INVALID, "window %d outside 1..%d", hp.window, kMaxWindow);
  if (hp.iterations < 1 || hp.iterations > kMaxIterations)
    return failf(SRS_ERR_INVALID, "iterations %d outside 1..%d", hp.iterations, kMaxIterations);
  if (hp.partitions < 1 || hp.partitions > kMaxPartitions)
    return failf(SRS_ERR_INVALID, "partitions %d outside 1..%d", hp.partitions, kMaxPartitions);
  return SRS_OK;
}

int i2v_check_ratings(const int32_t* user_id, const int32_t* movie_id, const int8_t* half, const int32_t* timestamp,
                      int64_t n_ratings, int32_t* n_slots) {
  PROPAGATE(check_ratings(user_id, movie_id, n_ratings, n_slots));
  if (n_ratings && (!half || !timestamp)) return failf(SRS_ERR_INVALID, "null ratings");
  const int n = (int)n_ratings;
  for (int i = 0; i < n; ++i) {
    if (half[i] < 1 || half[i] > 10)
      return failf(SRS_ERR_INVALID, "rating %d: %d half-stars is not a rating in [0.5, 5]", i, (int)half[i]);
    if (timestamp[i] <= 0) return failf(SRS_ERR_INVALID, "rating %d: timestamp %d is not positive", i, timestamp[i]);
  }
  if (n == 0) return failf(SRS_ERR_INVALID, "no ratings: the vocabulary would be empty");
  return SRS_OK;
}

int i2v_positive_corpus(HostCall& c, const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                        const int32_t* timestamp, int n, I2vCorpus* out) {
  Scratch& sc = c.sc;
  cudaStream_t s = c.s;
  int32_t *d_user, *d_movie, *d_ts, *d_order, *d_iota, *d_sel;
  uint32_t* d_suser;
  int8_t* d_half;
  uint8_t* d_flag;
  CUDA_TRY(sc.alloc(&d_user, n)); CUDA_TRY(sc.alloc(&d_movie, n)); CUDA_TRY(sc.alloc(&d_ts, n));
  CUDA_TRY(sc.alloc(&d_half, n)); CUDA_TRY(sc.alloc(&d_order, n)); CUDA_TRY(sc.alloc(&d_suser, n));
  CUDA_TRY(sc.alloc(&d_iota, n)); CUDA_TRY(sc.alloc(&d_sel, n)); CUDA_TRY(sc.alloc(&d_flag, n));
  CUDA_TRY(sc.alloc(&out->movie, n)); CUDA_TRY(sc.alloc(&out->user, n)); CUDA_TRY(sc.alloc(&out->n, 1));
  CUDA_TRY(cudaMemcpyAsync(d_user, user_id, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_movie, movie_id, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_ts, timestamp, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_half, half, n, cudaMemcpyHostToDevice, s));
  const int T = 256;
  PROPAGATE(user_time_order(s, d_user, d_ts, n, d_order, d_suser));
  i2v_flag_kernel<<<grid_for(n, T), T, 0, s>>>(d_order, d_half, n, d_flag, d_iota);
  LAUNCHED();
  CUB_RUN(c, cub::DeviceSelect::Flagged(tmp__, tb__, d_iota, d_flag, d_sel, out->n, n, s));
  i2v_gather_kernel<<<grid_for(n, T), T, 0, s>>>(d_sel, out->n, d_order, d_suser, d_movie, out->movie, out->user);
  LAUNCHED();
  return SRS_OK;
}

int word2vec_fit(HostCall& c, const int32_t* d_pmovie, const uint32_t* d_puser, const int* d_npos, int n,
                 int32_t n_slots, const srs_item2vec_params& hp, const char* what, int32_t capacity,
                 int32_t* vocab_ids, float* vectors, int32_t* vocab_size) {
  Scratch& sc = c.sc;
  cudaStream_t s = c.s;
  int32_t *d_count, *d_iota, *d_pword, *d_vidx, *d_words, *d_ustart, *d_offs, *d_points, *d_codelen;
  uint32_t *d_wuser, *d_code;
  uint8_t* d_flag;
  int* d_nsel;
  CUDA_TRY(sc.alloc(&d_count, n_slots)); CUDA_TRY(sc.alloc(&d_iota, n)); CUDA_TRY(sc.alloc(&d_flag, n));
  CUDA_TRY(sc.alloc(&d_nsel, 2));
  CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(int32_t) * n_slots, s));
  const int T = 256;
  i2v_count_kernel<<<grid_for(n, T), T, 0, s>>>(d_pmovie, d_npos, d_count);
  LAUNCHED();
  std::vector<int32_t> counts(n_slots);
  CUDA_TRY(cudaMemcpyAsync(counts.data(), d_count, sizeof(int32_t) * n_slots, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));

  // vocabulary: count >= minCount, count descending, ties by movie id ascending
  std::vector<int32_t> vocab;
  for (int32_t m = 0; m < n_slots; ++m)
    if (counts[m] >= kMinCount) vocab.push_back(m);
  std::stable_sort(vocab.begin(), vocab.end(), [&](int32_t x, int32_t y) { return counts[x] > counts[y]; });
  const int V = (int)vocab.size();
  if (V == 0) return failf(SRS_ERR_INVALID, "the vocabulary is empty: no movie has %d %s", kMinCount, what);
  if (V > capacity) return failf(SRS_ERR_RANGE, "vocabulary of %d words exceeds capacity %d", V, capacity);
  std::vector<int64_t> cn(V);
  std::vector<int32_t> vocab_index(n_slots, -1);
  int64_t train_words = 0;
  for (int w = 0; w < V; ++w) {
    cn[w] = counts[vocab[w]];
    vocab_index[vocab[w]] = w;
    train_words += cn[w];
  }
  std::vector<uint32_t> code_bits;
  std::vector<int32_t> points, codelen;
  const int deepest = huffman(cn, code_bits, points, codelen);
  if (deepest > kMaxCode)
    return failf(SRS_ERR_INVALID, "Huffman code of length %d: at most %d are supported", deepest, kMaxCode);
  std::vector<float> exp_table(kExpTable);
  for (int i = 0; i < kExpTable; ++i) {
    const double t = std::exp((2.0 * i / kExpTable - 1.0) * kMaxExp);
    exp_table[i] = (float)(t / (t + 1.0));
  }

  const int D = hp.vector_size, P = hp.partitions;
  const int nw = (int)train_words;
  const int64_t vd = (int64_t)V * D;
  float *d_exp, *d_syn0, *d_syn1, *d_l0 = nullptr, *d_l1 = nullptr;
  uint8_t *d_mod0 = nullptr, *d_mod1 = nullptr;
  CUDA_TRY(sc.alloc(&d_vidx, n_slots)); CUDA_TRY(sc.alloc(&d_pword, n)); CUDA_TRY(sc.alloc(&d_words, nw));
  CUDA_TRY(sc.alloc(&d_wuser, nw)); CUDA_TRY(sc.alloc(&d_ustart, nw)); CUDA_TRY(sc.alloc(&d_offs, nw));
  CUDA_TRY(sc.alloc(&d_points, (size_t)V * kMaxCode)); CUDA_TRY(sc.alloc(&d_codelen, V));
  CUDA_TRY(sc.alloc(&d_code, V)); CUDA_TRY(sc.alloc(&d_exp, kExpTable));
  CUDA_TRY(sc.alloc(&d_syn0, vd)); CUDA_TRY(sc.alloc(&d_syn1, vd));
  if (P > 1) {
    CUDA_TRY(sc.alloc(&d_l0, vd * P)); CUDA_TRY(sc.alloc(&d_l1, vd * P));
    CUDA_TRY(sc.alloc(&d_mod0, (size_t)V * P)); CUDA_TRY(sc.alloc(&d_mod1, (size_t)V * P));
  }
  CUDA_TRY(cudaMemcpyAsync(d_vidx, vocab_index.data(), sizeof(int32_t) * n_slots, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_points, points.data(), sizeof(int32_t) * points.size(), cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_codelen, codelen.data(), sizeof(int32_t) * V, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_code, code_bits.data(), sizeof(uint32_t) * V, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_exp, exp_table.data(), sizeof(float) * kExpTable, cudaMemcpyHostToDevice, s));

  // the in-vocabulary words and their sentence keys, then the sentence starts
  i2v_map_kernel<<<grid_for(n, T), T, 0, s>>>(d_pmovie, d_npos, n, d_vidx, d_pword, d_flag);
  LAUNCHED();
  CUB_RUN(c, cub::DeviceSelect::Flagged(tmp__, tb__, d_pword, d_flag, d_words, d_nsel + 1, n, s));
  CUB_RUN(c, cub::DeviceSelect::Flagged(tmp__, tb__, d_puser, d_flag, d_wuser, d_nsel + 1, n, s));
  i2v_user_start_kernel<<<grid_for(nw, T), T, 0, s>>>(d_wuser, nw, d_iota);
  LAUNCHED();
  CUB_RUN(c, cub::DeviceScan::InclusiveScan(tmp__, tb__, d_iota, d_ustart, MaxOp(), nw, s));
  i2v_chunk_kernel<<<grid_for(nw, T), T, 0, s>>>(d_ustart, nw, d_flag, d_iota);
  LAUNCHED();
  CUB_RUN(c, cub::DeviceSelect::Flagged(tmp__, tb__, d_iota, d_flag, d_offs, d_nsel, nw, s));

  i2v_init_kernel<<<grid_for(vd, T), T, 0, s>>>(d_syn0, vd, hp.seed, D);
  LAUNCHED();
  CUDA_TRY(cudaMemsetAsync(d_syn1, 0, sizeof(float) * vd, s));
  TrainArgs ta;
  ta.words = d_words; ta.chunk_offs = d_offs; ta.n_chunks = d_nsel; ta.n_words = nw;
  ta.code_bits = d_code; ta.points = d_points; ta.codelen = d_codelen; ta.exp_table = d_exp;
  ta.syn0 = P > 1 ? d_l0 : d_syn0; ta.syn1 = P > 1 ? d_l1 : d_syn1;   // one partition trains the tables in place
  ta.mod0 = d_mod0; ta.mod1 = d_mod1;
  ta.V = V; ta.D = D; ta.window = hp.window; ta.iterations = hp.iterations; ta.P = P;
  ta.seed = hp.seed; ta.train_words = train_words; ta.lr = kLearningRate;
  const int train_blocks = (P * 32 + 127) / 128;
  for (int k = 1; k <= hp.iterations; ++k) {
    if (P > 1) {
      i2v_broadcast_kernel<<<grid_for(vd * P, T), T, 0, s>>>(d_syn0, vd, P, d_l0);
      LAUNCHED();
      i2v_broadcast_kernel<<<grid_for(vd * P, T), T, 0, s>>>(d_syn1, vd, P, d_l1);
      LAUNCHED();
      CUDA_TRY(cudaMemsetAsync(d_mod0, 0, (size_t)V * P, s));
      CUDA_TRY(cudaMemsetAsync(d_mod1, 0, (size_t)V * P, s));
    }
    i2v_train_kernel<<<train_blocks, 128, 0, s>>>(ta, k);
    LAUNCHED();
    if (P > 1) {
      i2v_merge_kernel<<<grid_for(vd, T), T, 0, s>>>(d_l0, d_mod0, V, D, P, d_syn0);
      LAUNCHED();
      i2v_merge_kernel<<<grid_for(vd, T), T, 0, s>>>(d_l1, d_mod1, V, D, P, d_syn1);
      LAUNCHED();
    }
  }
  CUDA_TRY(cudaMemcpyAsync(vectors, d_syn0, sizeof(float) * vd, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  std::copy(vocab.begin(), vocab.end(), vocab_ids);
  *vocab_size = V;
  return SRS_OK;
}

}  // namespace srs

using namespace srs;

extern "C" int srs_item2vec_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                                 const int32_t* timestamp, int64_t n_ratings, const srs_item2vec_params* params,
                                 int32_t device, int32_t capacity, int32_t* vocab_ids, float* vectors,
                                 int32_t* vocab_size) {
  if (!vocab_size) return failf(SRS_ERR_INVALID, "null vocab_size");
  *vocab_size = 0;
  PROPAGATE(i2v_check_params(params));
  if (capacity < 0 || (capacity > 0 && (!vocab_ids || !vectors)))
    return failf(SRS_ERR_INVALID, "negative capacity or null outputs");
  int32_t n_slots = 0;
  PROPAGATE(i2v_check_ratings(user_id, movie_id, half, timestamp, n_ratings, &n_slots));

  HostCall c;
  PROPAGATE(c.begin(device));
  const int n = (int)n_ratings;
  I2vCorpus pos;
  PROPAGATE(i2v_positive_corpus(c, user_id, movie_id, half, timestamp, n, &pos));
  return word2vec_fit(c, pos.movie, pos.user, pos.n, n, n_slots, *params, "ratings >= 3.5", capacity, vocab_ids,
                      vectors, vocab_size);
}

extern "C" int srs_user_embeddings_host(const int32_t* user_id, const int32_t* movie_id, int64_t n_ratings,
                                        const int32_t* item_ids, const float* item_vectors, int32_t n_items,
                                        int32_t vector_size, int32_t device, int32_t capacity, int32_t* user_ids,
                                        float* user_vectors, int32_t* n_users) {
  if (!n_users) return failf(SRS_ERR_INVALID, "null n_users");
  *n_users = 0;
  if (vector_size < 1 || vector_size > kMaxDim)
    return failf(SRS_ERR_INVALID, "vector_size %d outside 1..%d", vector_size, kMaxDim);
  if (n_items < 0 || (n_items && (!item_ids || !item_vectors)))
    return failf(SRS_ERR_INVALID, "negative n_items or null items");
  if (capacity < 0 || (capacity > 0 && (!user_ids || !user_vectors)))
    return failf(SRS_ERR_INVALID, "negative capacity or null outputs");
  int32_t n_slots = 0;
  PROPAGATE(check_ratings(user_id, movie_id, n_ratings, &n_slots));
  for (int32_t i = 0; i < n_items; ++i) {
    if (item_ids[i] < 0 || item_ids[i] >= kMaxMovieSlots)
      return failf(SRS_ERR_INVALID, "item %d: id %d outside 0..2^24-1", i, item_ids[i]);
    n_slots = std::max(n_slots, item_ids[i] + 1);
  }
  std::vector<int32_t> row_of(std::max(n_slots, 1), -1);
  for (int32_t i = 0; i < n_items; ++i) {
    if (row_of[item_ids[i]] >= 0) return failf(SRS_ERR_INVALID, "item id %d appears twice", item_ids[i]);
    row_of[item_ids[i]] = i;
  }
  const int n = (int)n_ratings;
  if (n == 0) return SRS_OK;

  HostCall c;
  PROPAGATE(c.begin(device));
  Scratch& sc = c.sc;
  cudaStream_t s = c.s;
  const int D = vector_size;
  const size_t slots = row_of.size();
  int32_t *d_movie, *d_iota, *d_order, *d_uniq, *d_cnt, *d_start, *d_row;
  uint32_t *d_user, *d_suser;
  float *d_vec, *d_out;
  int* d_nu;
  CUDA_TRY(sc.alloc(&d_user, n)); CUDA_TRY(sc.alloc(&d_movie, n)); CUDA_TRY(sc.alloc(&d_iota, n));
  CUDA_TRY(sc.alloc(&d_order, n)); CUDA_TRY(sc.alloc(&d_suser, n)); CUDA_TRY(sc.alloc(&d_uniq, n));
  CUDA_TRY(sc.alloc(&d_cnt, n)); CUDA_TRY(sc.alloc(&d_start, n)); CUDA_TRY(sc.alloc(&d_row, slots));
  CUDA_TRY(sc.alloc(&d_vec, (size_t)std::max(n_items, 1) * D)); CUDA_TRY(sc.alloc(&d_out, (size_t)n * D));
  CUDA_TRY(sc.alloc(&d_nu, 1));
  std::vector<int32_t> iota(n);
  for (int i = 0; i < n; ++i) iota[i] = i;
  CUDA_TRY(cudaMemcpyAsync(d_user, user_id, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_movie, movie_id, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_iota, iota.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_row, row_of.data(), sizeof(int32_t) * slots, cudaMemcpyHostToDevice, s));
  if (n_items)
    CUDA_TRY(cudaMemcpyAsync(d_vec, item_vectors, sizeof(float) * n_items * D, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemsetAsync(d_cnt, 0, sizeof(int32_t) * n, s));
  // a stable sort by user: each user's ratings stay in file order
  CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_user, d_suser, d_iota, d_order, n, 0, 31, s));
  CUB_RUN(c, cub::DeviceRunLengthEncode::Encode(tmp__, tb__, d_suser, d_uniq, d_cnt, d_nu, n, s));
  CUB_RUN(c, cub::DeviceScan::ExclusiveSum(tmp__, tb__, d_cnt, d_start, n, s));
  i2v_user_kernel<<<(int)(((int64_t)n * 32 + 127) / 128), 128, 0, s>>>(d_order, d_start, d_cnt, d_nu, d_movie, d_row,
                                                                     d_vec, D, d_out);
  LAUNCHED();
  int nu = 0;
  CUDA_TRY(cudaMemcpyAsync(&nu, d_nu, sizeof(int), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  if (nu > capacity) return failf(SRS_ERR_RANGE, "%d users exceed capacity %d", nu, capacity);
  CUDA_TRY(cudaMemcpyAsync(user_ids, d_uniq, sizeof(int32_t) * nu, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(user_vectors, d_out, sizeof(float) * nu * D, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  *n_users = nu;
  return SRS_OK;
}
