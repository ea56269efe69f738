// hostcall.h - what the host entry points share: error reporting (failf and the CUDA_TRY / LAUNCHED / PROPAGATE
// macros), the launch grid and counter hash of the offline jobs, and HostCall, the device, stream, allocations and
// CUB storage of one offline call (DESIGN.md section 5).  Then the offline jobs' functions that cross files.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <vector>

#include "../../include/srs_ctr.h"
#include "kernels.h"

namespace srs {

// model.cu: format the message srs_last_error() reports on this thread; returns `code`
int failf(int code, const char* fmt, ...);
// model.cu: SRS_OK when `device` is one of this machine's CUDA devices (the current device is not changed)
int check_device(int device);

// return SRS_ERR_CUDA from the calling function when a CUDA runtime (or CUB) call fails
#define CUDA_TRY(expr)                                                                                          \
  do {                                                                                                          \
    cudaError_t e__ = (expr);                                                                                   \
    if (e__ != cudaSuccess)                                                                                     \
      return ::srs::failf(SRS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__,      \
                          __LINE__);                                                                            \
  } while (0)

// after each kernel launch of the library's own: count it, and report a launch that was refused
#define LAUNCHED()                        \
  do {                                    \
    ++::srs::g_launch_count;              \
    CUDA_TRY(cudaGetLastError());         \
  } while (0)

// return a non-zero SRS_* code from the calling function (the callee has set the message)
#define PROPAGATE(expr)                   \
  do {                                    \
    const int rc__ = (expr);              \
    if (rc__ != SRS_OK) return rc__;      \
  } while (0)

// The most blocks a grid-stride kernel over n elements is launched with: 64 per SM of the H100's 132, a few
// waves of resident blocks, so that the grid stays small and in range however large n is
constexpr int kMaxGridBlocks = 132 * 64;
inline int grid_for(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  return (int)(b < 1 ? 1 : b > kMaxGridBlocks ? kMaxGridBlocks : b);
}

// The library's counter-based hash: splitmix64's finaliser of x + (i + 1) * golden.  srs_fill_uniform,
// collab.random_split, item2vec's initial vectors and window draws, the random walks, ALS's initial factors and the
// sample split all draw from it; oracle/als_c.c, oracle/item2vec_c.c and the Python oracles restate it.
__host__ __device__ __forceinline__ uint64_t splitmix(uint64_t x, uint64_t i) {
  uint64_t z = x + (i + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// a uniform in [0, 1): the top 53 bits of splitmix(key, i) over 2^53
__host__ __device__ __forceinline__ double uniform53(uint64_t key, uint64_t i) {
  return (double)(splitmix(key, i) >> 11) * 0x1p-53;
}

struct Scratch {                       // device allocations of one host call, freed when it ends
  std::vector<void*> ptrs;
  ~Scratch() { for (void* p : ptrs) cudaFree(p); }
  template <class T>
  cudaError_t alloc(T** p, size_t count) {
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, (count ? count : 1) * sizeof(T));
    if (e == cudaSuccess) ptrs.push_back(q);
    *p = static_cast<T*>(q);
    return e;
  }
};

// One offline host call: its device, its stream, its allocations and CUB's temporary storage.  An entry point checks
// its arguments, then begin(), then works on `s` and copies out; whichever way it returns, the stream is
// synchronised and destroyed first and the allocations are freed after.
struct HostCall {
  Scratch sc;
  cudaStream_t s = nullptr;
  void* cub_tmp = nullptr;             // CUB's temporary storage (CUB_RUN), grown as the calls ask
  size_t cub_bytes = 0;
  HostCall() = default;
  HostCall(const HostCall&) = delete;
  HostCall& operator=(const HostCall&) = delete;
  ~HostCall() {                        // `sc` frees after this body
    if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
  }
  // the first CUDA call of an entry point: every argument check comes before it
  int begin(int32_t device) {
    PROPAGATE(check_device(device));
    CUDA_TRY(cudaSetDevice(device));
    CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    return SRS_OK;
  }
  // *d = a device copy of h[0 .. count), in stream order
  template <class T>
  int upload(T** d, const T* h, size_t count) {
    CUDA_TRY(sc.alloc(d, count));
    if (count) CUDA_TRY(cudaMemcpyAsync(*d, h, sizeof(T) * count, cudaMemcpyHostToDevice, s));
    return SRS_OK;
  }
  cudaError_t cub_need(size_t bytes) {
    if (bytes <= cub_bytes) return cudaSuccess;
    uint8_t* q = nullptr;
    const cudaError_t e = sc.alloc(&q, bytes);
    cub_tmp = q;
    cub_bytes = e == cudaSuccess ? bytes : 0;
    return e;
  }
};

// CUB's two calls - the size query, then the work - of a device-wide primitive on the call `hc`; write the
// primitive's first two arguments as tmp__, tb__
#define CUB_RUN(hc, call_with_tmp)                                                                             \
  do {                                                                                                          \
    size_t need__ = 0;                                                                                          \
    { void* tmp__ = nullptr; size_t& tb__ = need__; CUDA_TRY(call_with_tmp); }                                  \
    CUDA_TRY((hc).cub_need(need__));                                                                            \
    { void* tmp__ = (hc).cub_tmp; size_t tb__ = (hc).cub_bytes; CUDA_TRY(call_with_tmp); }                      \
  } while (0)

// ---- featureeng.cu ---------------------------------------------------------------------------------------------
// The (user, timestamp string, file index) order of n ratings (device arrays), as the reference's jobs order a
// user's ratings: d_order[i] = file index of the i-th, d_user_sorted[i] = its user.  Stable radix sorts on `s`;
// temporaries are stream-ordered allocations.  Returns an SRS_* code.
int user_time_order(cudaStream_t s, const int32_t* d_user, const int32_t* d_ts, int n, int32_t* d_order,
                    uint32_t* d_user_sorted);
// The movies' exact integer moments of n ratings (device arrays): d_mmom[3 m .. 3 m + 2] += count, sum h, sum h^2 of
// movie m's half-stars (64-bit integer atomics; the caller zeroes d_mmom); d_iota[i] = i.
cudaError_t launch_movie_moments(const int32_t* d_movie, const int8_t* d_half, int n, int32_t* d_iota,
                                 unsigned long long* d_mmom, cudaStream_t s);

// ---- item2vec.cu: the Embedding job's sentences and Word2Vec, shared with graphemb.cu ---------------------------
// Each returns an SRS_* code and sets the last error message.
int i2v_check_params(const srs_item2vec_params* params);
// the ratings' checks of srs_item2vec_host (ids, half-stars, timestamps, at least one rating); *n_slots = max movie + 1
int i2v_check_ratings(const int32_t* user_id, const int32_t* movie_id, const int8_t* half, const int32_t* timestamp,
                      int64_t n_ratings, int32_t* n_slots);
struct I2vCorpus {                     // device: *n words, movie[i] in sentence order, user[i] its sentence's key
  int32_t* movie;
  uint32_t* user;
  int* n;
};
// processItemSequence: the n ratings (host) uploaded, and their positives (>= 3.5) grouped by user ascending, each
// user's in (timestamp string, input index) order; arrays of n entries allocated in `c`
int i2v_positive_corpus(HostCall& c, const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                        const int32_t* timestamp, int n, I2vCorpus* out);
// Word2Vec.fit over the device corpus of *d_n <= n words (movie ids < n_slots) whose sentences are the runs of
// equal keys: vocabulary, Huffman tree, exp table, the 1000-word cut and training; the outputs as srs_item2vec_host.
// `what` names the words in the empty-vocabulary message.  Synchronises c.s.
int word2vec_fit(HostCall& c, const int32_t* d_words, const uint32_t* d_keys, const int* d_n, int n, int32_t n_slots,
                 const srs_item2vec_params& hp, const char* what, int32_t capacity, int32_t* vocab_ids,
                 float* vectors, int32_t* vocab_size);

// ---- similar.cu and model.cu: what recforyou.cu reads of a catalogue and of a model (no copies) --------------------
struct SimilarCatalogView {
  int32_t device, n_movies, dim;
  bool hash_order;                     // getMovies' order is known (no HashMap bin treeified)
  const int32_t* movie_id;             // [n_movies] by load-order slot
  const float* emb;                    // [n_emb][dim] movie vectors
  const int32_t* emb_row;              // [n_movies] the movie's row of emb, -1 for none
  int32_t n_rec;                       // entries of rec
  const int32_t* rec;                  // getMovies(800, "rating"): slots, in that order
};
SimilarCatalogView similar_catalog_view(const srs_similar_catalog* h);
struct ModelView {
  int32_t kind, device;                // srs_spec.kind and the model's device
  const NcfParams* ncf;                // the placed NeuralCF / two-tower weights (other kinds: unset)
  int32_t hist_cols;                   // history columns the forward reads: T (DIN, DIEN), 1 (W&D) or 0
  int32_t n_users, n_movies;           // the model's id vocabularies
  const void* movie_feats;             // srs_model_set_movie_features' table, [movie_feats_rows][8 words]; or null
  int32_t movie_feats_rows;
};
ModelView model_view(const srs_model* m);
// The model's own forward, as its predict calls run it: the kernel the model chose at creation, on `s`.  The caller
// holds model_mutex(m) from before it reads the movie table until its last launch has finished.
std::mutex& model_mutex(srs_model* m);
size_t model_batch_bytes(const srs_model* m, size_t B);   // the packed batch of B rows (model.cu's slot layout)
// the view of a packed batch of B rows at `block`, its scores to `probs` and its range errors to `err_flag`
BatchView model_batch_view(const srs_model* m, uint8_t* block, size_t B, float* probs, int* err_flag);
int model_launch(srs_model* m, const BatchView& v, cudaStream_t s);

}  // namespace srs
