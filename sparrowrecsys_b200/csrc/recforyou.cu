// recforyou.cu - the reference's "Recommended for you" page, RecForYouProcess.getRecList(userId, size, model)
// (online/recprocess/RecForYouProcess.java:29-105), for many users per call.  DESIGN.md section 4.25 gives the
// semantics; oracle/recforyou.py restates the Java.
//
// User table (srs_recforyou_users_create_host, once): the distinct user ids of ratings.csv (DataManager.userMap) by
//   a radix sort and a unique pass, and each user's row of the userEmb.csv vectors (rfy_emb_row_kernel: the last line
//   of a user wins, lines of unknown users are skipped).
// Candidates: getMovies(800, "rating"), which the similar-movies catalogue keeps in rating order (similar.cu).
// Query (srs_recforyou_host), one block per user after one pass over the candidates:
//   default   score candidates.size() - i: the candidate order itself, no sort;
//   emb       rfy_candidates_kernel forms each candidate's squared norm once per call (one warp each, the sum
//             cosine.cuh forms), rfy_rank_kernel the dot of every (user, candidate) pair and the cosine;
//   nerualcf  rfy_ncf_items_kernel runs each candidate's item side once per call - NeuralCF's b0 + W0_item . m, the
//             first half of ncf_kernel's first-layer FMA chain, or the two-tower item tower - and
//             rfy_ncf_users_kernel each user's tower; rfy_ncf_kernel finishes each pair as ncf_kernel does (the
//             user half of the chain, the hidden layers and the output; or the dot and the final Dense), so every
//             score has ncf_kernel's bits for that (user, movie) row;
//   order     a bitonic sort in shared memory by (desc_key(score), movie id): Double.compare descending, NaN first,
//             ties by movie id (similar.cu's rule).
// A user outside the model's vocabulary, or any candidate outside it (latched by rfy_ncf_items_kernel, read as row
// 0), makes the user's status SRS_RECFORYOU_MODEL_RANGE with an empty list.  No float atomics and every sum in a
// fixed order: the same inputs give the same bits.
// "nerualcf" with every other model (srs_recforyou_ctr_host, DESIGN.md section 4.26): the users' uf: records
//   (srs_recforyou_users_set_features_host) and the model's movie table.  rfy_ctr_status_kernel applies predict's
//   range rule per user; the users that pass go in chunks of kCtrBatchBytes of assembled rows through
//   rfy_ctr_requests_kernel (srs_rank_user_host's request block per user), util.cu's assemble_request_kernel, the
//   model's own forward launch and rfy_ctr_sort_kernel (the order above).
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "../../include/srs_ctr.h"
#include "cosine.cuh"
#include "double_key.cuh"
#include "hostcall.h"
#include "ncf_layers.cuh"

struct srs_recforyou_users {
  int32_t device = 0;
  int32_t n_users = 0, dim = 0;
  int32_t* ids = nullptr;                // [n_users] the distinct user ids, ascending
  int32_t* emb_row = nullptr;            // [n_users] the user's row of emb, -1 for none
  float* emb = nullptr;                  // [n_emb][dim]
  int32_t* feat = nullptr;               // srs_recforyou_users_set_features_host: [n_users][kFeatWords], or null
  ~srs_recforyou_users() {
    cudaSetDevice(device);
    for (void* p : {(void*)ids, (void*)emb_row, (void*)emb, (void*)feat}) cudaFree(p);
  }
};

namespace srs {
namespace {

constexpr int kT = 256;                  // threads of the per-user kernels and of the grid-stride ones
constexpr int kItemT = 128;              // threads of rfy_ncf_items_kernel / rfy_ncf_users_kernel
constexpr uint64_t kPad = ~0ull;         // an empty sort entry: after every real one
// A user's `uf:` record in the user table: userGenre1..5 (vocabulary index, -1 missing), userAvgRating,
// userRatingCount, userRatingStddev (float bits), userRatedMovie1..5 in key order
constexpr int kFeatWords = 13;
constexpr int kGenres = 19;              // the reference's genre vocabulary (srs_spec.n_genres)
// The CTR page's assembled batch (the forward's packed rows of one chunk of users x the candidates) stays within
// this many bytes; the chunk is as many users as fit, at least one
constexpr size_t kCtrBatchBytes = (size_t)256 << 20;

#define RFY_GRID_STRIDE(i, n) \
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// position of `id` in the ascending ids[0 .. n), -1 when absent
__device__ __forceinline__ int find_id(const int32_t* __restrict__ ids, int n, int32_t id) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ids[mid] < id) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && ids[lo] == id ? lo : -1;
}

// DataManager.loadUserEmb sets each known user's vector in file order, so the last line of a user wins
__global__ void rfy_emb_row_kernel(const int32_t* __restrict__ emb_user, int n_emb, const int32_t* __restrict__ ids,
                                   int n_users, int32_t* __restrict__ emb_row) {
  RFY_GRID_STRIDE(i, n_emb) {
    const int u = find_id(ids, n_users, emb_user[i]);
    if (u >= 0) atomicMax(emb_row + u, (int32_t)i);
  }
}

struct Cands {                           // the call's candidates, getMovies(800, "rating") order
  int n;
  int32_t* id;                           // [n] movie ids
  int32_t* row;                          // [n] the movie's vector row, -1 for none
  double* n2;                            // [n] emb: the squared norm of that vector
};

// one warp per candidate: its id, its vector row and (emb) the vector's squared norm
__global__ void rfy_candidates_kernel(SimilarCatalogView cat, int with_norm, Cands c) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x / 32);
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; i < c.n; i += warps) {
    const int slot = cat.rec[i];
    const int r = cat.emb_row[slot];
    if (with_norm && r >= 0) {
      const float* v = cat.emb + (size_t)r * cat.dim;
      const double n2 = warp_product_sum(v, v, cat.dim, lane);
      if (lane == 0) c.n2[i] = n2;
    }
    if (lane == 0) {
      c.id[i] = cat.movie_id[slot];
      c.row[i] = r;
    }
  }
}

struct Out {                             // one call's device outputs, `width` entries per user
  int32_t* ids;
  double* scores;
  int32_t* count;
  int32_t* status;
  int width;
};

// the user's table position, or its status (and an empty list) when getUserById finds nobody
__device__ __forceinline__ int user_or_status(const int32_t* __restrict__ ids, int n_users, int32_t uid, int q,
                                              const Out& o) {
  const int u = find_id(ids, n_users, uid);
  if (u < 0 && threadIdx.x == 0) {
    o.count[q] = 0;
    o.status[q] = SRS_RECFORYOU_UNKNOWN_USER;
  }
  return u;
}

__device__ __forceinline__ bool item_greater(const ulonglong2& a, const ulonglong2& b) {
  return a.x > b.x || (a.x == b.x && a.y > b.y);
}

// item[i] = (desc_key(score of candidate i), (movie id ^ 2^31) << 32 | i) for i < n, padded to np (a power of two):
// sort ascending - score descending, ties by movie id - and write the first min(n, width) as user q's list
__device__ void sort_and_write(ulonglong2* item, int n, int np, int q, const Out& o) {
  const int tid = threadIdx.x;
  for (int i = n + tid; i < np; i += blockDim.x) item[i] = make_ulonglong2(kPad, kPad);
  __syncthreads();
  for (int w = 2; w <= np; w <<= 1)
    for (int j = w >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < np / 2; t += blockDim.x) {
        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1)), hi = lo | j;
        const ulonglong2 x = item[lo], y = item[hi];
        if (item_greater(x, y) == ((lo & w) == 0)) {
          item[lo] = y;
          item[hi] = x;
        }
      }
      __syncthreads();
    }
  const int n_out = n < o.width ? n : o.width;
  for (int r = tid; r < n_out; r += blockDim.x) {
    o.ids[(size_t)q * o.width + r] = (int32_t)((uint32_t)(item[r].y >> 32) ^ 0x80000000u);
    o.scores[(size_t)q * o.width + r] = key_score(item[r].x);
  }
  if (tid == 0) {
    o.count[q] = n_out;
    o.status[q] = SRS_RECFORYOU_OK;
  }
}

__device__ __forceinline__ ulonglong2 make_item(double score, int32_t movie_id, int i) {
  return make_ulonglong2(desc_key(score), ((uint64_t)((uint32_t)movie_id ^ 0x80000000u) << 32) | (uint32_t)i);
}

struct UserTable {
  const int32_t *ids, *emb_row;
  const float* emb;
  int n_users, dim;
  const int32_t* feat;                   // [n_users][kFeatWords] (the CTR page only)
};

// The emb and default rankers, one block per user.  default: candidates.size() - i, already in order.  emb:
// calculateEmbSimilarScore, -1 without a user vector, a movie vector or equal dimensions; one warp per candidate.
__global__ void __launch_bounds__(kT)
rfy_rank_kernel(UserTable ut, SimilarCatalogView cat, Cands c, int emb, int np, const int32_t* __restrict__ query,
                Out o) {
  extern __shared__ ulonglong2 item[];
  const int q = blockIdx.x, tid = threadIdx.x;
  const int u = user_or_status(ut.ids, ut.n_users, query[q], q, o);
  if (u < 0) return;
  if (!emb) {
    const int n_out = c.n < o.width ? c.n : o.width;
    for (int r = tid; r < n_out; r += kT) {
      o.ids[(size_t)q * o.width + r] = c.id[r];
      o.scores[(size_t)q * o.width + r] = (double)(c.n - r);
    }
    if (tid == 0) {
      o.count[q] = n_out;
      o.status[q] = SRS_RECFORYOU_OK;
    }
    return;
  }
  const int urow = ut.emb_row[u];
  const bool scored = urow >= 0 && ut.dim == cat.dim;
  if (!scored) {
    for (int i = tid; i < c.n; i += kT) item[i] = make_item(-1.0, c.id[i], i);
  } else {
    const int warp = tid >> 5, lane = tid & 31;
    const float* uv = ut.emb + (size_t)urow * ut.dim;
    const double n1 = warp_product_sum(uv, uv, ut.dim, lane);
    for (int i = warp; i < c.n; i += kT / 32) {
      const int r = c.row[i];
      double s = -1.0;                   // Embedding.calculateSimilarity of a missing vector
      if (r >= 0) s = cosine_value(warp_product_sum(uv, cat.emb + (size_t)r * cat.dim, cat.dim, lane), n1, c.n2[i]);
      if (lane == 0) item[i] = make_item(s, c.id[i], i);
    }
  }
  __syncthreads();
  sort_and_write(item, c.n, np, q, o);
}

// ---- "nerualcf": the served NeuralCF / two-tower model ------------------------------------------------------------
// The candidates' item side, one thread each: NeuralCF's first-layer bias and item rows (ncf_kernel's
// first_layer_accum over the item row, which it runs before the user row), or the two-tower item tower.  A movie
// id outside the model latches *err and is read as row 0, as checked_id does.
template <int EP, int HP>
__global__ void __launch_bounds__(kItemT)
rfy_ncf_items_kernel(NcfParams p, Cands c, float* __restrict__ part, int* __restrict__ err) {
  extern __shared__ __align__(16) float sw[];
  for (int i = threadIdx.x; i < p.blob_floats; i += blockDim.x) sw[i] = __ldg(p.blob + i);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.n) return;
  const int mid = checked_id(c.id[i], p.n_movies, err);
  const float* mrow = p.movie + (size_t)mid * EP;
  float h[HP];
#pragma unroll
  for (int j = 0; j < HP; ++j) h[j] = sw[p.b_off[0] + j];
  first_layer_accum<EP, HP>(h, mrow, sw + p.w_off[0]);
  if (p.two_towers) {
#pragma unroll
    for (int j = 0; j < HP; ++j) h[j] = fmaxf(h[j], 0.f);
    for (int l = 1; l < p.n_layers; ++l) hidden_layer<HP>(h, sw + p.w_off[l], sw + p.b_off[l]);
  }
#pragma unroll
  for (int j = 0; j < HP; ++j) part[(size_t)i * HP + j] = h[j];
}

// two towers: each in-range user's tower, one thread per user of the call
template <int EP, int HP>
__global__ void __launch_bounds__(kItemT)
rfy_ncf_users_kernel(NcfParams p, const int32_t* __restrict__ query, int n, float* __restrict__ tower) {
  extern __shared__ __align__(16) float sw[];
  for (int i = threadIdx.x; i < p.blob_floats; i += blockDim.x) sw[i] = __ldg(p.blob + i);
  __syncthreads();
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const int uid = query[q];
  if ((unsigned)uid >= (unsigned)p.n_users) return;
  float h[HP];
#pragma unroll
  for (int j = 0; j < HP; ++j) h[j] = sw[p.b_off[3] + j];
  first_layer_accum<EP, HP>(h, p.user + (size_t)uid * EP, sw + p.w_off[3]);
#pragma unroll
  for (int j = 0; j < HP; ++j) h[j] = fmaxf(h[j], 0.f);
  for (int l = 1; l < p.n_layers; ++l) hidden_layer<HP>(h, sw + p.w_off[3 + l], sw + p.b_off[3 + l]);
#pragma unroll
  for (int j = 0; j < HP; ++j) tower[(size_t)q * HP + j] = h[j];
}

// One block per user, one thread per (user, candidate) pair: the rest of ncf_kernel's row, then the sort
template <int EP, int HP>
__global__ void __launch_bounds__(kT)
rfy_ncf_kernel(NcfParams p, UserTable ut, Cands c, const float* __restrict__ part, const float* __restrict__ tower,
               const int* __restrict__ err, int np, const int32_t* __restrict__ query, Out o) {
  extern __shared__ __align__(16) unsigned char smem[];
  ulonglong2* item = reinterpret_cast<ulonglong2*>(smem);
  float* sw = reinterpret_cast<float*>(smem + sizeof(ulonglong2) * np);
  const int q = blockIdx.x, tid = threadIdx.x;
  const int uid = query[q];
  if (user_or_status(ut.ids, ut.n_users, uid, q, o) < 0) return;
  if ((unsigned)uid >= (unsigned)p.n_users || *err) {    // TF-Serving rejects the request
    if (tid == 0) {
      o.count[q] = 0;
      o.status[q] = SRS_RECFORYOU_MODEL_RANGE;
    }
    return;
  }
  for (int i = tid; i < p.blob_floats; i += kT) sw[i] = __ldg(p.blob + i);
  __syncthreads();
  for (int i = tid; i < c.n; i += kT) {
    float s;
    if (!p.two_towers) {
      float h[HP];
#pragma unroll
      for (int j = 0; j < HP; ++j) h[j] = part[(size_t)i * HP + j];
      first_layer_accum<EP, HP>(h, p.user + (size_t)uid * EP, sw + p.w_off[0] + EP * HP);   // then user rows
#pragma unroll
      for (int j = 0; j < HP; ++j) h[j] = fmaxf(h[j], 0.f);
      for (int l = 1; l < p.n_layers; ++l) hidden_layer<HP>(h, sw + p.w_off[l], sw + p.b_off[l]);
      float z = sw[p.out_b];
#pragma unroll
      for (int j = 0; j < HP; ++j) z = fmaf(h[j], sw[p.out_w + j], z);
      s = sigmoidf_acc(z);
    } else {
      const float* hi = part + (size_t)i * HP;
      const float* hu = tower + (size_t)q * HP;
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < HP; ++j) d = fmaf(hi[j], hu[j], d);
      s = p.final_dense ? sigmoidf_acc(fmaf(d, sw[p.out_w], sw[p.out_b])) : d;
    }
    item[i] = make_item((double)s, c.id[i], i);
  }
  __syncthreads();
  sort_and_write(item, c.n, np, q, o);
}

template <int EP, int HP>
int launch_ncf_t(const NcfParams& p, const UserTable& ut, const Cands& c, const int32_t* query, int n, int np,
                 float* part, float* tower, int* err, const Out& o, cudaStream_t s) {
  const size_t wbytes = sizeof(float) * p.blob_floats;
  if (c.n) {
    rfy_ncf_items_kernel<EP, HP><<<(c.n + kItemT - 1) / kItemT, kItemT, wbytes, s>>>(p, c, part, err);
    LAUNCHED();
  }
  if (p.two_towers) {
    rfy_ncf_users_kernel<EP, HP><<<(n + kItemT - 1) / kItemT, kItemT, wbytes, s>>>(p, query, n, tower);
    LAUNCHED();
  }
  const size_t smem = sizeof(ulonglong2) * np + wbytes;
  CUDA_TRY(cudaFuncSetAttribute(rfy_ncf_kernel<EP, HP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  rfy_ncf_kernel<EP, HP><<<n, kT, smem, s>>>(p, ut, c, part, tower, err, np, query, o);
  LAUNCHED();
  return SRS_OK;
}

int launch_rfy_ncf(const NcfParams& p, const UserTable& ut, const Cands& c, const int32_t* query, int n, int np,
               float* part, float* tower, int* err, const Out& o, cudaStream_t s) {
#define RFY_NCF_CASE(E_, H_) \
  if (p.EP == E_ && p.HP == H_) return launch_ncf_t<E_, H_>(p, ut, c, query, n, np, part, tower, err, o, s);
  RFY_NCF_CASE(12, 16) RFY_NCF_CASE(16, 16) RFY_NCF_CASE(32, 16) RFY_NCF_CASE(64, 16)
  RFY_NCF_CASE(12, 32) RFY_NCF_CASE(16, 32) RFY_NCF_CASE(32, 32) RFY_NCF_CASE(64, 32)
#undef RFY_NCF_CASE
  return failf(SRS_ERR_INVALID, "recommend for you: no kernel for padded width %d and hidden width %d", p.EP, p.HP);
}

// ---- "nerualcf" with every other served model: the uf: / mf: features (DESIGN.md section 4.26) -------------------
// How the model reads ids: which positions hold the stored userRatedMovie1..5 and how a movie id is range-checked
struct CtrReads {
  int n_users, n_movies, n_table;        // the model's vocabularies; the rows of its movie table
  int hc;                                // history columns of a row
  int pos[5];                            // the position of userRatedMovie<k + 1> among them, -1 when not read
  int f32_ids;                           // DIN, DIEN: movie ids pass through float32 before the check
};

__device__ __forceinline__ bool movie_in_model(int id, const CtrReads& r) {
  if (r.f32_ids) id = __float2int_rz(__int2float_rn(id));
  return static_cast<unsigned>(id) < static_cast<unsigned>(r.n_movies);
}

// srs_recforyou_users_set_features_host: the user's record from its last row (rows of unknown ids skipped), or the
// defaults of an empty hash
__global__ void rfy_feat_row_kernel(const int32_t* __restrict__ uid, int n, const int32_t* __restrict__ ids,
                                    int n_users, int32_t* __restrict__ row) {
  RFY_GRID_STRIDE(i, n) {
    const int u = find_id(ids, n_users, uid[i]);
    if (u >= 0) atomicMax(row + u, (int32_t)i);
  }
}

__global__ void rfy_feat_kernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ row, int n_users,
                                int32_t* __restrict__ feat) {
  RFY_GRID_STRIDE(i, (int64_t)n_users * kFeatWords) {
    const int u = (int)(i / kFeatWords), w = (int)(i - (int64_t)u * kFeatWords);
    const int r = row[u];
    feat[i] = r >= 0 ? rows[(size_t)r * kFeatWords + w] : (w < 5 ? -1 : 0);
  }
}

// Each queried user's status before any forward: UNKNOWN_USER outside the table; MODEL_RANGE when its userId, a
// history id the model reads or any candidate (outside the model or past its movie table) would make predict
// reject its rows; else pass[q] = 1 and the forward scores it
__global__ void __launch_bounds__(kT)
rfy_ctr_status_kernel(UserTable ut, Cands c, CtrReads r, const int32_t* __restrict__ query, int n, Out o,
                      int32_t* __restrict__ pass) {
  bool bad = false;
  for (int i = threadIdx.x; i < c.n; i += kT) {
    const int id = c.id[i];
    bad |= !movie_in_model(id, r) || static_cast<unsigned>(id) >= static_cast<unsigned>(r.n_table);
  }
  const bool bad_cands = __syncthreads_or(bad);
  RFY_GRID_STRIDE(q, n) {
    const int32_t uid = query[q];
    const int u = find_id(ut.ids, ut.n_users, uid);
    int st = SRS_RECFORYOU_UNKNOWN_USER;
    if (u >= 0) {
      bool ok = !bad_cands && static_cast<unsigned>(uid) < static_cast<unsigned>(r.n_users);
      for (int k = 0; k < 5; ++k)
        if (r.pos[k] >= 0) ok = ok && movie_in_model(ut.feat[(size_t)u * kFeatWords + 8 + k], r);
      st = ok ? SRS_RECFORYOU_OK : SRS_RECFORYOU_MODEL_RANGE;
    }
    pass[q] = st == SRS_RECFORYOU_OK;
    if (st != SRS_RECFORYOU_OK) {
      o.count[q] = 0;
      o.status[q] = st;
    }
  }
}

// One warp per user of the chunk: its request record for launch_assemble_request, srs_rank_user_host's block
// [userId | userGenre1..5 | 3 numerics | hist[hc]] with the stored history ids at their positions and 0 elsewhere
__global__ void __launch_bounds__(kT)
rfy_ctr_requests_kernel(UserTable ut, CtrReads r, const int32_t* __restrict__ query, const int32_t* __restrict__ sel,
                        int n, int32_t* __restrict__ req) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (kT / 32);
  const int words = 9 + r.hc;
  for (int64_t j = ((int64_t)blockIdx.x * kT + threadIdx.x) / 32; j < n; j += warps) {
    const int32_t uid = query[sel[j]];
    const int u = find_id(ut.ids, ut.n_users, uid);
    const int32_t* f = ut.feat + (size_t)u * kFeatWords;
    int32_t* out = req + (size_t)j * words;
    for (int w = lane; w < words; w += 32) {
      int32_t v = 0;
      if (w == 0) v = uid;
      else if (w < 9) v = f[w - 1];
      else
        for (int k = 0; k < 5; ++k)
          if (r.pos[k] == w - 9) v = f[8 + k];
      out[w] = v;
    }
  }
}

// One block per user of the chunk: its candidates' forward scores, widened to double, in the page's order
__global__ void __launch_bounds__(kT)
rfy_ctr_sort_kernel(const float* __restrict__ probs, Cands c, int np, const int32_t* __restrict__ sel, Out o) {
  extern __shared__ ulonglong2 item[];
  const int j = blockIdx.x;
  const float* p = probs + (size_t)j * c.n;
  for (int i = threadIdx.x; i < c.n; i += kT) item[i] = make_item((double)p[i], c.id[i], i);
  __syncthreads();
  sort_and_write(item, c.n, np, sel[j], o);
}

template <class T>
int persist(T** p, size_t count) {       // a user-table allocation, freed by its destructor
  CUDA_TRY(cudaMalloc(p, (count ? count : 1) * sizeof(T)));
  return SRS_OK;
}

int create_users(const int32_t* rating_user, int64_t n_ratings, const int32_t* emb_user, const float* emb,
                 int32_t n_emb, int32_t dim, int32_t device, srs_recforyou_users** out) {
  if (!out) return failf(SRS_ERR_INVALID, "user table: null output handle");
  *out = nullptr;
  if (n_ratings < 0 || n_ratings > INT32_MAX)
    return failf(SRS_ERR_INVALID, "user table: n_ratings %lld outside 0 .. 2^31 - 1", (long long)n_ratings);
  if (n_ratings > 0 && !rating_user) return failf(SRS_ERR_INVALID, "user table: null rating_user");
  if (n_emb < 0 || dim < 0) return failf(SRS_ERR_INVALID, "user table: n_emb %d or dim %d < 0", n_emb, dim);
  if (n_emb > 0 && (dim < 1 || !emb_user || !emb))
    return failf(SRS_ERR_INVALID, "user table: %d vectors need dim >= 1 (got %d), emb_user and emb", n_emb, dim);

  HostCall c;
  PROPAGATE(c.begin(device));
  srs_recforyou_users* h = new (std::nothrow) srs_recforyou_users;
  if (!h) return failf(SRS_ERR_NOMEM, "user table: out of host memory");
  std::unique_ptr<srs_recforyou_users> owner(h);
  h->device = device;
  h->dim = n_emb > 0 ? dim : 0;
  const int nr = (int)n_ratings;

  // DataManager.userMap: every user id of a rating line
  int32_t *d_user, *d_sorted, *d_unique;
  int* d_n;
  PROPAGATE(c.upload(&d_user, rating_user, (size_t)nr));
  CUDA_TRY(c.sc.alloc(&d_sorted, (size_t)nr));
  CUDA_TRY(c.sc.alloc(&d_unique, (size_t)nr));
  CUDA_TRY(c.sc.alloc(&d_n, 1));
  int n_users = 0;
  if (nr) {
    CUB_RUN(c, cub::DeviceRadixSort::SortKeys(tmp__, tb__, d_user, d_sorted, nr, 0, 32, c.s));
    CUB_RUN(c, cub::DeviceSelect::Unique(tmp__, tb__, d_sorted, d_unique, d_n, nr, c.s));
    CUDA_TRY(cudaMemcpyAsync(&n_users, d_n, sizeof(int), cudaMemcpyDeviceToHost, c.s));
    CUDA_TRY(cudaStreamSynchronize(c.s));
  }
  h->n_users = n_users;
  PROPAGATE(persist(&h->ids, n_users));
  PROPAGATE(persist(&h->emb_row, n_users));
  if (n_users)
    CUDA_TRY(cudaMemcpyAsync(h->ids, d_unique, sizeof(int32_t) * n_users, cudaMemcpyDeviceToDevice, c.s));
  CUDA_TRY(cudaMemsetAsync(h->emb_row, 0xFF, sizeof(int32_t) * (n_users ? n_users : 1), c.s));

  // userEmb.csv
  if (n_emb > 0) {
    PROPAGATE(persist(&h->emb, (size_t)n_emb * dim));
    CUDA_TRY(cudaMemcpyAsync(h->emb, emb, sizeof(float) * (size_t)n_emb * dim, cudaMemcpyHostToDevice, c.s));
    int32_t* d_eid;
    PROPAGATE(c.upload(&d_eid, emb_user, n_emb));
    if (n_users) {
      rfy_emb_row_kernel<<<grid_for(n_emb, kT), kT, 0, c.s>>>(d_eid, n_emb, h->ids, n_users, h->emb_row);
      LAUNCHED();
    }
  }
  CUDA_TRY(cudaStreamSynchronize(c.s));
  *out = owner.release();
  return SRS_OK;
}

int recommend(const srs_similar_catalog* catalog, const srs_recforyou_users* users, const srs_model* model,
              int32_t ranker, const int32_t* user_ids, int32_t n, int32_t size, int32_t* out_ids,
              double* out_scores, int32_t* out_count, int32_t* out_status) {
  if (n < 0) return failf(SRS_ERR_INVALID, "recommend for you: n_users %d < 0", n);
  if (size < 1) return failf(SRS_ERR_INVALID, "recommend for you: size %d < 1", size);
  if (ranker != SRS_RECFORYOU_DEFAULT && ranker != SRS_RECFORYOU_EMB && ranker != SRS_RECFORYOU_NEURALCF)
    return failf(SRS_ERR_INVALID, "recommend for you: unknown ranker %d", ranker);
  if (!catalog || !users) return failf(SRS_ERR_INVALID, "recommend for you: null catalog or user table");
  const SimilarCatalogView cat = similar_catalog_view(catalog);
  if (!cat.hash_order)
    return failf(SRS_ERR_INVALID, "recommend for you: a HashMap bin of the movie ids is treeified (9 or more ids in "
                 "one bucket of a table of 64 or more), so getMovies' order of ties is not load order within a bucket");
  if (users->device != cat.device)
    return failf(SRS_ERR_INVALID, "recommend for you: the user table is on device %d, the catalogue on device %d",
                 users->device, cat.device);
  const NcfParams* ncf = nullptr;
  if (ranker == SRS_RECFORYOU_NEURALCF) {
    if (!model) return failf(SRS_ERR_INVALID, "recommend for you: the nerualcf ranker needs a model");
    const ModelView mv = model_view(model);
    if (mv.kind != SRS_NEURALCF && mv.kind != SRS_TWOTOWERS)
      return failf(SRS_ERR_INVALID, "recommend for you: the nerualcf ranker needs a NeuralCF or two-tower model, "
                   "not kind %d", mv.kind);
    if (mv.device != cat.device)
      return failf(SRS_ERR_INVALID, "recommend for you: the model is on device %d, the catalogue on device %d",
                   mv.device, cat.device);
    ncf = mv.ncf;
  }
  if (n > 0 && (!user_ids || !out_ids || !out_scores || !out_count || !out_status))
    return failf(SRS_ERR_INVALID, "recommend for you: null user or output array");
  if (n == 0) return SRS_OK;
  const size_t Q = (size_t)n;
  memset(out_ids, 0, sizeof(int32_t) * Q * size);
  memset(out_scores, 0, sizeof(double) * Q * size);

  const int nc = cat.n_rec;
  int np = 32;
  while (np < nc) np <<= 1;
  const int width = std::max(1, std::min(size, nc));
  HostCall c;
  PROPAGATE(c.begin(cat.device));
  int32_t *d_query;
  Out o;
  o.width = width;
  PROPAGATE(c.upload(&d_query, user_ids, Q));
  CUDA_TRY(c.sc.alloc(&o.ids, Q * width));
  CUDA_TRY(c.sc.alloc(&o.scores, Q * width));
  CUDA_TRY(c.sc.alloc(&o.count, Q));
  CUDA_TRY(c.sc.alloc(&o.status, Q));
  CUDA_TRY(cudaMemsetAsync(o.ids, 0, sizeof(int32_t) * Q * width, c.s));
  CUDA_TRY(cudaMemsetAsync(o.scores, 0, sizeof(double) * Q * width, c.s));
  Cands cd{nc, nullptr, nullptr, nullptr};
  CUDA_TRY(c.sc.alloc(&cd.id, nc));
  CUDA_TRY(c.sc.alloc(&cd.row, nc));
  CUDA_TRY(c.sc.alloc(&cd.n2, nc));
  if (nc) {
    rfy_candidates_kernel<<<(nc + kT / 32 - 1) / (kT / 32), kT, 0, c.s>>>(cat, ranker == SRS_RECFORYOU_EMB, cd);
    LAUNCHED();
  }
  const UserTable ut{users->ids, users->emb_row, users->emb, users->n_users, users->dim};
  if (ranker != SRS_RECFORYOU_NEURALCF) {
    const size_t smem = sizeof(ulonglong2) * np;
    CUDA_TRY(cudaFuncSetAttribute(rfy_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rfy_rank_kernel<<<n, kT, smem, c.s>>>(ut, cat, cd, ranker == SRS_RECFORYOU_EMB, np, d_query, o);
    LAUNCHED();
  } else {
    float *d_part, *d_tower;
    int* d_err;
    CUDA_TRY(c.sc.alloc(&d_part, (size_t)nc * ncf->HP));
    CUDA_TRY(c.sc.alloc(&d_tower, ncf->two_towers ? Q * ncf->HP : 1));
    CUDA_TRY(c.sc.alloc(&d_err, 1));
    CUDA_TRY(cudaMemsetAsync(d_err, 0, sizeof(int), c.s));
    PROPAGATE(launch_rfy_ncf(*ncf, ut, cd, d_query, n, np, d_part, d_tower, d_err, o, c.s));
  }
  CUDA_TRY(cudaMemcpy2DAsync(out_ids, sizeof(int32_t) * size, o.ids, sizeof(int32_t) * width,
                             sizeof(int32_t) * width, Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpy2DAsync(out_scores, sizeof(double) * size, o.scores, sizeof(double) * width,
                             sizeof(double) * width, Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(out_count, o.count, sizeof(int32_t) * Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(out_status, o.status, sizeof(int32_t) * Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));
  return SRS_OK;
}

int set_user_features(srs_recforyou_users* users, int32_t n, const int32_t* user_id, const int32_t* user_genre,
                      const float* user_numerics, const int32_t* hist) {
  if (n < 0) return failf(SRS_ERR_INVALID, "user features: n %d < 0", n);
  if (n > 0 && (!user_id || !user_genre || !user_numerics || !hist))
    return failf(SRS_ERR_INVALID, "user features: null user_id, user_genre, user_numerics or hist");
  if (!users) return failf(SRS_ERR_INVALID, "user features: null user table");
  std::vector<int32_t> rows((size_t)n * kFeatWords);
  for (int i = 0; i < n; ++i) {
    int32_t* r = rows.data() + (size_t)i * kFeatWords;
    for (int g = 0; g < 5; ++g) {
      const int32_t v = user_genre[(size_t)i * 5 + g];
      if (v >= kGenres)
        return failf(SRS_ERR_RANGE, "user features: row %d, genre index %d outside the vocabulary of %d", i, v, kGenres);
      r[g] = v < 0 ? -1 : v;
    }
    memcpy(r + 5, user_numerics + (size_t)i * 3, 12);
    memcpy(r + 8, hist + (size_t)i * 5, 20);
  }
  HostCall c;
  PROPAGATE(c.begin(users->device));
  const int nu = users->n_users;
  int32_t *d_rows, *d_uid, *d_row, *feat = nullptr;
  PROPAGATE(c.upload(&d_rows, rows.data(), rows.size()));
  PROPAGATE(c.upload(&d_uid, user_id, (size_t)n));
  CUDA_TRY(c.sc.alloc(&d_row, (size_t)nu));
  CUDA_TRY(cudaMemsetAsync(d_row, 0xFF, sizeof(int32_t) * (nu ? nu : 1), c.s));
  CUDA_TRY(cudaMalloc(&feat, sizeof(int32_t) * ((size_t)nu * kFeatWords + 1)));
  std::unique_ptr<int32_t, decltype(&cudaFree)> owner(feat, &cudaFree);
  if (n > 0 && nu > 0) {
    rfy_feat_row_kernel<<<grid_for(n, kT), kT, 0, c.s>>>(d_uid, n, users->ids, nu, d_row);
    LAUNCHED();
  }
  if (nu > 0) {
    rfy_feat_kernel<<<grid_for((int64_t)nu * kFeatWords, kT), kT, 0, c.s>>>(d_rows, d_row, nu, feat);
    LAUNCHED();
  }
  CUDA_TRY(cudaStreamSynchronize(c.s));
  cudaFree(users->feat);
  users->feat = owner.release();
  return SRS_OK;
}

// the positions of userRatedMovie1..5 among the model's history inputs, as rank_user places them: DIN and DIEN
// read history_keys(T), the T keys userRatedMovie1..T in ASCII order; W&D reads userRatedMovie1; the rest none
void history_positions(const ModelView& mv, int T, int pos[5]) {
  for (int k = 0; k < 5; ++k) pos[k] = -1;
  if (mv.kind == SRS_WIDENDEEP) pos[0] = mv.hist_cols > 0 ? 0 : -1;
  if (mv.kind != SRS_DIN && mv.kind != SRS_DIEN) return;
  std::vector<std::string> keys;
  for (int k = 1; k <= T; ++k) keys.push_back("userRatedMovie" + std::to_string(k));
  std::sort(keys.begin(), keys.end());
  for (int p = 0; p < T && p < mv.hist_cols; ++p)
    for (int k = 1; k <= 5; ++k)
      if (keys[p] == "userRatedMovie" + std::to_string(k)) pos[k - 1] = p;
}

int recommend_ctr(const srs_similar_catalog* catalog, const srs_recforyou_users* users, srs_model* model,
                  const int32_t* user_ids, int32_t n, int32_t size, int32_t* out_ids, double* out_scores,
                  int32_t* out_count, int32_t* out_status) {
  if (n < 0) return failf(SRS_ERR_INVALID, "recommend for you: n_users %d < 0", n);
  if (size < 1) return failf(SRS_ERR_INVALID, "recommend for you: size %d < 1", size);
  if (n > 0 && (!user_ids || !out_ids || !out_scores || !out_count || !out_status))
    return failf(SRS_ERR_INVALID, "recommend for you: null user or output array");
  if (!model) return failf(SRS_ERR_INVALID, "recommend for you: null model");
  const ModelView mv = model_view(model);
  if (mv.kind == SRS_NEURALCF || mv.kind == SRS_TWOTOWERS)      // (userId, movieId) only: srs_recforyou_host
    return recommend(catalog, users, model, SRS_RECFORYOU_NEURALCF, user_ids, n, size, out_ids, out_scores,
                     out_count, out_status);
  if (!catalog || !users) return failf(SRS_ERR_INVALID, "recommend for you: null catalog or user table");
  const SimilarCatalogView cat = similar_catalog_view(catalog);
  if (!cat.hash_order)
    return failf(SRS_ERR_INVALID, "recommend for you: a HashMap bin of the movie ids is treeified (9 or more ids in "
                 "one bucket of a table of 64 or more), so getMovies' order of ties is not load order within a bucket");
  if (users->device != cat.device || mv.device != cat.device)
    return failf(SRS_ERR_INVALID, "recommend for you: the user table is on device %d, the model on device %d, the "
                 "catalogue on device %d", users->device, mv.device, cat.device);
  if (!users->feat)
    return failf(SRS_ERR_INVALID, "recommend for you: this model reads the users' uf: features: call "
                 "srs_recforyou_users_set_features_host first");
  std::lock_guard<std::mutex> lock(model_mutex(model));
  const ModelView m = model_view(model);          // the movie table, read under the model's lock
  if (!m.movie_feats)
    return failf(SRS_ERR_INVALID, "recommend for you: this model reads movie features: call "
                 "srs_model_set_movie_features first");
  if (n == 0) return SRS_OK;
  const size_t Q = (size_t)n;
  memset(out_ids, 0, sizeof(int32_t) * Q * size);
  memset(out_scores, 0, sizeof(double) * Q * size);

  CtrReads r{};
  r.n_users = m.n_users;
  r.n_movies = m.n_movies;
  r.n_table = m.movie_feats_rows;
  r.hc = m.hist_cols;
  r.f32_ids = m.kind == SRS_DIN || m.kind == SRS_DIEN;
  history_positions(m, m.hist_cols, r.pos);
  const int nc = cat.n_rec;
  int np = 32;
  while (np < nc) np <<= 1;
  const int width = std::max(1, std::min(size, nc));
  HostCall c;
  PROPAGATE(c.begin(cat.device));
  int32_t *d_query, *d_pass, *d_sel;
  int *d_nsel, *d_err;
  Out o;
  o.width = width;
  PROPAGATE(c.upload(&d_query, user_ids, Q));
  CUDA_TRY(c.sc.alloc(&o.ids, Q * width));
  CUDA_TRY(c.sc.alloc(&o.scores, Q * width));
  CUDA_TRY(c.sc.alloc(&o.count, Q));
  CUDA_TRY(c.sc.alloc(&o.status, Q));
  CUDA_TRY(c.sc.alloc(&d_pass, Q));
  CUDA_TRY(c.sc.alloc(&d_sel, Q));
  CUDA_TRY(c.sc.alloc(&d_nsel, 1));
  CUDA_TRY(c.sc.alloc(&d_err, 1));
  CUDA_TRY(cudaMemsetAsync(o.ids, 0, sizeof(int32_t) * Q * width, c.s));
  CUDA_TRY(cudaMemsetAsync(o.scores, 0, sizeof(double) * Q * width, c.s));
  CUDA_TRY(cudaMemsetAsync(d_err, 0, sizeof(int), c.s));
  Cands cd{nc, nullptr, nullptr, nullptr};
  CUDA_TRY(c.sc.alloc(&cd.id, nc));
  CUDA_TRY(c.sc.alloc(&cd.row, nc));
  CUDA_TRY(c.sc.alloc(&cd.n2, nc));
  if (nc) {
    rfy_candidates_kernel<<<(nc + kT / 32 - 1) / (kT / 32), kT, 0, c.s>>>(cat, 0, cd);
    LAUNCHED();
  }
  const UserTable ut{users->ids, users->emb_row, users->emb, users->n_users, users->dim, users->feat};
  rfy_ctr_status_kernel<<<grid_for(n, kT), kT, 0, c.s>>>(ut, cd, r, d_query, n, o, d_pass);
  LAUNCHED();
  // the users that passed, in query order
  CUB_RUN(c, cub::DeviceSelect::Flagged(tmp__, tb__, thrust::counting_iterator<int32_t>(0), d_pass, d_sel,
                                        d_nsel, n, c.s));
  int n_sel = 0;
  CUDA_TRY(cudaMemcpyAsync(&n_sel, d_nsel, sizeof(int), cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));

  // chunks of users whose assembled rows fit kCtrBatchBytes: requests, assembly, the model's forward, the order
  const size_t user_bytes = model_batch_bytes(model, (size_t)nc);
  const int chunk = n_sel == 0 ? 0 : (int)std::max<size_t>(1, std::min<size_t>(n_sel, user_bytes ? kCtrBatchBytes /
                                                                                user_bytes : n_sel));
  if (chunk > 0) {
    const size_t rows = (size_t)chunk * nc;
    uint8_t* block;
    float* probs;
    int32_t* req;
    CUDA_TRY(c.sc.alloc(&block, model_batch_bytes(model, rows) + 256));
    CUDA_TRY(c.sc.alloc(&probs, rows));
    CUDA_TRY(c.sc.alloc(&req, (size_t)chunk * (9 + r.hc)));
    const size_t smem = sizeof(ulonglong2) * np;
    CUDA_TRY(cudaFuncSetAttribute(rfy_ctr_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int j0 = 0; j0 < n_sel; j0 += chunk) {
      const int k = std::min(chunk, n_sel - j0);
      if (nc) {
        rfy_ctr_requests_kernel<<<grid_for((int64_t)k * 32, kT), kT, 0, c.s>>>(ut, r, d_query, d_sel + j0, k, req);
        LAUNCHED();
        const BatchView v = model_batch_view(model, block, (size_t)k * nc, probs, d_err);
        CUDA_TRY(launch_assemble_request(req, k, cd.id, nc, m.movie_feats, m.movie_feats_rows, r.hc, 1,
                                         const_cast<int32_t*>(v.movie_id), const_cast<int32_t*>(v.user_id),
                                         const_cast<int32_t*>(v.hist), const_cast<int32_t*>(v.movie_genre),
                                         const_cast<int32_t*>(v.user_genre), const_cast<float*>(v.numerics), d_err,
                                         c.s));
        PROPAGATE(model_launch(model, v, c.s));
      }
      rfy_ctr_sort_kernel<<<k, kT, smem, c.s>>>(probs, cd, np, d_sel + j0, o);
      LAUNCHED();
    }
  }
  int err = 0;
  CUDA_TRY(cudaMemcpyAsync(&err, d_err, sizeof(int), cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpy2DAsync(out_ids, sizeof(int32_t) * size, o.ids, sizeof(int32_t) * width,
                             sizeof(int32_t) * width, Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpy2DAsync(out_scores, sizeof(double) * size, o.scores, sizeof(double) * width,
                             sizeof(double) * width, Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(out_count, o.count, sizeof(int32_t) * Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(out_status, o.status, sizeof(int32_t) * Q, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));
  if (err)        // the status kernel admits only rows that the forward accepts: this is a library bug
    return failf(SRS_ERR_RANGE, "recommend for you: an id passed the page's range checks but not the forward's");
  return SRS_OK;
}

}  // namespace
}  // namespace srs

extern "C" int srs_recforyou_users_create_host(const int32_t* rating_user, int64_t n_ratings,
                                               const int32_t* emb_user, const float* emb, int32_t n_emb,
                                               int32_t dim, int32_t device, srs_recforyou_users** out) {
  return srs::create_users(rating_user, n_ratings, emb_user, emb, n_emb, dim, device, out);
}

extern "C" void srs_recforyou_users_destroy(srs_recforyou_users* users) { delete users; }

extern "C" int srs_recforyou_host(const srs_similar_catalog* catalog, const srs_recforyou_users* users,
                                  const srs_model* model, int32_t ranker, const int32_t* user_ids, int32_t n_users,
                                  int32_t size, int32_t* out_ids, double* out_scores, int32_t* out_count,
                                  int32_t* out_status) {
  return srs::recommend(catalog, users, model, ranker, user_ids, n_users, size, out_ids, out_scores, out_count,
                        out_status);
}

extern "C" int srs_recforyou_users_set_features_host(srs_recforyou_users* users, int32_t n, const int32_t* user_id,
                                                     const int32_t* user_genre, const float* user_numerics,
                                                     const int32_t* hist) {
  return srs::set_user_features(users, n, user_id, user_genre, user_numerics, hist);
}

extern "C" int srs_recforyou_ctr_host(const srs_similar_catalog* catalog, const srs_recforyou_users* users,
                                      srs_model* model, const int32_t* user_ids, int32_t n_users, int32_t size,
                                      int32_t* out_ids, double* out_scores, int32_t* out_count, int32_t* out_status) {
  return srs::recommend_ctr(catalog, users, model, user_ids, n_users, size, out_ids, out_scores, out_count,
                            out_status);
}
