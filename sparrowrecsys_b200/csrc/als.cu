// als.cu - the reference's CollaborativeFiltering job (Spark ML ALS, explicit or implicit feedback) on one device:
// the factors from double-precision normal equations solved by Cholesky, the fused top-k recommendations and the
// ranking metrics that score them.  DESIGN.md sections 4.13 and 4.17 give the semantics, the orders Spark leaves
// open and the bounds.
//
// srs_als_fit_host, on one stream, inputs uploaded once:
//   1. four stable radix sorts: by user and by movie (the dense, ascending ids: run-length encodings), then the
//      user-ordered ratings by movie - the by-movie layout (movie, user, input order) - and that by user - the
//      by-user layout (user, movie, input order);
//   2. als_gather_kernel: each layout's counterpart index and rating; each side's entities sorted longest first;
//   -- the ids come to the host once: the users' initial factors are drawn there (O(users * rank)) --
//   3. per iteration, with no host round trip: als_solve_kernel over the movies, then over the users.
// als_solve_kernel runs one block per entity, longest first.  The block stages 32 of the entity's ratings at a time
// in shared memory; each thread owns elements of the packed upper ata and of atb and adds each rating's term to
// them in rating order (dspr / daxpy).  Then thread c owns column c: row r of the Cholesky factor is computed in
// step r (dpptrf's elements, each in its own order), then the two triangular solves (dpptrs).  Every double
// operation is an explicitly rounded intrinsic and there are no atomics on data: the same inputs give the same
// bits as oracle/als_c.c.  A non-positive or NaN pivot latches (half-step, entity) in an error word (atomicMin:
// the first half-step, then the lowest entity).
//
// srs_als_fit_folds_host (DESIGN.md section 4.15) fits up to 64 models - each its own rank, max_iter, reg_param and
// excluded fold - over one rating set: the layouts of steps 1-2 once, each rating's fold gathered into both, then one
// als_solve_kernel<true> launch per half-step for every model.  A fold's subset of a layout keeps its order, so
// each model's results are bit for bit srs_als_fit_host's on its training ratings.
//
// srs_als_fit_implicit_host (DESIGN.md section 4.17) is the same fit with Spark's implicitPrefs: before each
// half-step als_yty_kernel sums YtY over the source factors in Spark's ten blocks (entity id mod 10, ascending id;
// one block of elements per thread slice, each element owned by one thread), als_yty_merge_kernel adds the blocks
// in block order, and als_solve_kernel<false, true> starts each entity's ata from YtY and adds each rating's
// confidence and preference terms.
//
// srs_als_fit_nonnegative_host and srs_als_fit_folds_nonnegative_host (DESIGN.md section 4.21) are these fits with
// Spark's nonnegative = true: als_solve_kernel<..., true> keeps the accumulation and replaces the Cholesky tail by
// NNLS.solve on one warp (nnls_warp); a batched fit launches its NNLS models over their own slice of the model list.
//
// srs_ranking_metrics_host: RankingMetrics' per-query precision@k, NDCG@k and average precision, one warp per
// query (ranking_metrics_kernel), over each query's labels sorted on the device; the means on the host.
//
// als_recommend_kernel (srs_als_recommend_host): 32 sources per block, 4 per warp; destinations stream through
// shared memory in tiles of 128, transposed so that each lane reads its own 4.  Each lane computes 4 x 4 exact
// sequential float dots (__fmul_rn / __fadd_rn from 0.0f, no fma); the warp keeps a sorted list of `num` per
// source, inserting a candidate only when it beats the list's last entry.  The top-k under a strict total order
// does not depend on the order candidates arrive in.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"

namespace srs {
namespace {

constexpr int kMaxRank = 64;           // one thread per factor column
constexpr int kMaxNum = 128;           // four list entries per lane
constexpr int64_t kMaxRatings = 21000000;
constexpr int kMaxModels = 64;         // models of one batched fit
constexpr int kMaxFolds = 65536;
constexpr int kSolveThreads = 128;
constexpr int kChunk = 32;             // ratings staged per step of the accumulation
constexpr int kRecWarps = 8;
constexpr int kSrcPerWarp = 4;
constexpr int kSrcPerBlock = kRecWarps * kSrcPerWarp;
constexpr int kTile = 128;             // destinations per shared-memory tile, 4 per lane
constexpr unsigned kFull = 0xffffffffu;
constexpr int kYtyBlocks = 10;         // Spark's default number of ALS blocks
constexpr int kYtyThreads = 128;       // packed YtY elements per thread slice
constexpr int kRankWarps = 8;          // queries per block of ranking_metrics_kernel

// The initial factor of the user with id `user`: `rank` draws of java.util.Random.nextGaussian's polar method on
// uniforms uniform53(splitmix(seed, user), c), each cast to float, then scaled by
// 1.0f / snrm2 (reference BLAS's scaled sum of squares).  oracle/als_c.c restates this function line for line.
void init_factor(uint64_t seed, int32_t user, int rank, float* out) {
  const uint64_t key = splitmix(seed, (uint64_t)(uint32_t)user);
  uint64_t c = 0;
  for (int d = 0; d < rank; d += 2) {
    double v1, v2, s;
    do {
      v1 = 2 * uniform53(key, c++) - 1;
      v2 = 2 * uniform53(key, c++) - 1;
      s = v1 * v1 + v2 * v2;
    } while (s >= 1 || s == 0);
    const double m = std::sqrt(-2 * std::log(s) / s);
    out[d] = (float)(v1 * m);
    if (d + 1 < rank) out[d + 1] = (float)(v2 * m);
  }
  float scale = 0.0f, ssq = 1.0f;
  for (int d = 0; d < rank; ++d) {
    if (out[d] == 0.0f) continue;
    const float a = std::fabs(out[d]);
    if (scale < a) {
      const float t = scale / a;
      ssq = 1.0f + ssq * (t * t);
      scale = a;
    } else {
      const float t = a / scale;
      ssq = ssq + t * t;
    }
  }
  const float inv = 1.0f / (scale * std::sqrt(ssq));
  for (int d = 0; d < rank; ++d) out[d] = out[d] * inv;
}

__global__ void als_iota_kernel(int32_t* __restrict__ out, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = i;
}

// head[p] = 1 where the sorted key changes (the first rating of an entity)
__global__ void als_head_kernel(const int32_t* __restrict__ key, int n, int32_t* __restrict__ head) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    head[i] = (i == 0 || key[i] != key[i - 1]) ? 1 : 0;
}

// dense[perm[p]] = seg[p] - 1 (seg: the inclusive sum of the heads)
__global__ void als_scatter_kernel(const int32_t* __restrict__ perm, const int32_t* __restrict__ seg, int n,
                                   int32_t* __restrict__ dense) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dense[perm[i]] = seg[i] - 1;
}

// key[p] = dense[perm[p]]
__global__ void als_key_kernel(const int32_t* __restrict__ perm, const int32_t* __restrict__ dense, int n,
                               int32_t* __restrict__ key) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) key[i] = dense[perm[i]];
}

// a layout's counterpart (source) index and rating, in layout order
__global__ void als_gather_kernel(const int32_t* __restrict__ perm, const int32_t* __restrict__ src_dense,
                                  const float* __restrict__ rating, int n, int32_t* __restrict__ src,
                                  float* __restrict__ r) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int q = perm[i];
    src[i] = src_dense[q];
    r[i] = rating[q];
  }
}

struct Side {
  const int32_t* off;                  // [nE + 1] first rating of each entity in the layout
  const int32_t* src;                  // [n] counterpart index of each rating, in accumulation order
  const float* r;                      // [n] its rating
  const int32_t* order;                // [nE] entities, longest first
  int nE;
};

// One model of a batched fit (srs_als_fit_folds_host)
struct BatchModel {
  int k;
  int half_steps;                      // 2 * max_iter
  double reg;
  int exclude;                         // the fold whose ratings it skips; -1: none
  size_t user_off, movie_off;          // its [nU][k] user and [nM][k] movie factors in the shared arrays
};

struct Batch {
  const BatchModel* models;            // [M]
  const int32_t* fold;                 // [n] fold of each rating, in the side's layout order
  int32_t* count;                      // [M][nE] each entity's training ratings in each model
  int M;
  bool to_users;                       // this half-step solves the users from the movies
};

// The implicit-feedback settings of a half-step (srs_als_fit_implicit_host)
struct Implicit {
  const double* yty;                   // [k (k + 1) / 2] packed YtY of the source factors
  double alpha;
};

// NNLS.solve's wall test: step dir(i) > x(i) (1 - 1e-14)
constexpr double kWallShrink = 1.0 - 1e-14;

// element (i, j) of the symmetric matrix whose upper triangle is the packed P
__device__ __forceinline__ double nnls_sym(const double* P, int i, int j) {
  return i <= j ? P[j * (j + 1) / 2 + i] : P[i * (i + 1) / 2 + j];
}

// row i of dgemv "N" (y = A v, beta 0): from 0, columns j ascending with v(j) != 0, y += (1.0 v(j)) A(i,j)
__device__ __forceinline__ double nnls_row(const double* P, const double* v, int i, int k) {
  double y = 0.0;
  for (int j = 0; j < k; ++j) {
    const double vj = v[j];
    if (vj != 0.0) y = __dadd_rn(y, __dmul_rn(vj, nnls_sym(P, i, j)));
  }
  return y;
}

// NNLS.solve's stop(step, ndir, nx)
__device__ __forceinline__ bool nnls_stop(double step, double ndir, double nx) {
  return step != step || step < 1e-7 || step > 1e40 || ndir < __dmul_rn(1e-12, nx) || ndir < 1e-32;
}

// Spark's NNLS.solve(ata, atb) on one warp (DESIGN.md section 4.21): P the packed upper ata with lambda on its
// diagonal, B atb, ws [5][k] doubles of shared scratch; out [k] = x(i).toFloat.  Lane t owns rows t and t + 32 of x,
// res, grad and dir.  The vectors the sums read are published in ws; every lane runs each sequential sum (ddot
// from 0, i ascending) and the step-7 scan over them, so the scalars are the same on every lane and need no
// broadcast.  Each operation is one explicitly rounded intrinsic.
__device__ void nnls_warp(const double* P, const double* B, double* ws, int k, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  double* sx = ws;                                      // x
  double* sg = ws + k;                                  // grad
  double* sd = ws + 2 * k;                              // dir
  double* sr = ws + 3 * k;                              // res
  double* sa = ws + 4 * k;                              // A grad, then A dir
  double x[2], b[2], ld[2], g[2], d[2];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int i = lane + 32 * q;
    x[q] = ld[q] = g[q] = d[q] = 0.0;
    b[q] = i < k ? B[i] : 0.0;
    if (i < k) sx[i] = 0.0;
  }
  const int iter_max = max(400, 20 * k);
  double last_norm = 0.0;
  int iterno = 0, last_wall = 0;
  __syncwarp();
  while (iterno < iter_max) {
    // res = A x - atb; grad = res, zero where it points out of the orthant at a bound
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = lane + 32 * q;
      if (i < k) {
        const double res = __dsub_rn(nnls_row(P, sx, i, k), b[q]);
        g[q] = res > 0.0 && x[q] == 0.0 ? 0.0 : res;
        sr[i] = res;
        sg[i] = g[q];
      }
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 2; ++q)
      if (lane + 32 * q < k) sa[lane + 32 * q] = nnls_row(P, sg, lane + 32 * q, k);
    __syncwarp();
    double ngrad = 0.0, top = 0.0, den = 0.0, nx = 0.0;   // ddot(grad, grad), ddot(grad, res), ddot(A grad, grad), ddot(x, x)
    for (int j = 0; j < k; ++j) {
      const double gj = sg[j], xj = sx[j];
      ngrad = __dadd_rn(ngrad, __dmul_rn(gj, gj));
      top = __dadd_rn(top, __dmul_rn(gj, sr[j]));
      den = __dadd_rn(den, __dmul_rn(sa[j], gj));
      nx = __dadd_rn(nx, __dmul_rn(xj, xj));
    }
    double step = __ddiv_rn(top, __dadd_rn(den, 1e-20));
    double ndir = ngrad;                                // ddot(grad, grad) again, the same bits
    bool cg = false;
    if (iterno > last_wall + 1) {                       // the conjugate direction dir = grad + (ngrad / lastNorm) lastDir
      const double alpha = __ddiv_rn(ngrad, last_norm);
      __syncwarp();                                     // sa is read
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int i = lane + 32 * q;
        if (i < k) {
          d[q] = alpha != 0.0 ? __dadd_rn(g[q], __dmul_rn(alpha, ld[q])) : g[q];   // daxpy returns for alpha 0
          sd[i] = d[q];
        }
      }
      __syncwarp();
#pragma unroll
      for (int q = 0; q < 2; ++q)
        if (lane + 32 * q < k) sa[lane + 32 * q] = nnls_row(P, sd, lane + 32 * q, k);
      __syncwarp();
      double top2 = 0.0, den2 = 0.0, nd = 0.0;
      for (int j = 0; j < k; ++j) {
        const double dj = sd[j];
        top2 = __dadd_rn(top2, __dmul_rn(dj, sr[j]));
        den2 = __dadd_rn(den2, __dmul_rn(sa[j], dj));
        nd = __dadd_rn(nd, __dmul_rn(dj, dj));
      }
      const double dstep = __ddiv_rn(top2, __dadd_rn(den2, 1e-20));
      if (!nnls_stop(dstep, nd, nx)) {
        step = dstep;
        ndir = nd;
        cg = true;
      }
    }
    if (nnls_stop(step, ndir, nx)) break;
    __syncwarp();                                       // sd is read
    if (!cg)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int i = lane + 32 * q;
        d[q] = g[q];
        if (i < k) sd[i] = g[q];
      }
    __syncwarp();
    for (int j = 0; j < k; ++j) {                       // don't run through the walls: in order, each j sees the step
      const double dj = sd[j], xj = sx[j];              // the ones before it left
      if (__dmul_rn(step, dj) > xj) step = __ddiv_rn(xj, dj);
    }
    bool wall = false;
#pragma unroll
    for (int q = 0; q < 2; ++q)
      if (lane + 32 * q < k) {
        const double sdv = __dmul_rn(step, d[q]);
        if (sdv > __dmul_rn(x[q], kWallShrink)) {
          x[q] = 0.0;
          wall = true;
        } else {
          x[q] = __dsub_rn(x[q], sdv);
        }
      }
    if (__any_sync(kFull, wall)) last_wall = iterno;
    __syncwarp();                                       // sx is read
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (lane + 32 * q < k) sx[lane + 32 * q] = x[q];
      ld[q] = d[q];
    }
    last_norm = ngrad;
    ++iterno;
    __syncwarp();
  }
#pragma unroll
  for (int q = 0; q < 2; ++q)
    if (lane + 32 * q < k) out[lane + 32 * q] = __double2float_rn(x[q]);
}

// One block per entity (the blockIdx.x-th longest; batched: block b is model b % M's (b / M)-th longest entity):
// NormalEquation.add over its ratings, then CholeskySolver.solve(ne, n * regParam) (dppsv "U": dpptrf, then
// dpptrs's two dtpsv).  A batched model skips its excluded fold's ratings, so its n counts the rest; an entity with
// none is not in that model and its block writes nothing but the count.  Implicit: ata starts as YtY, each rating
// adds dspr(c1) and, when positive, daxpy(1 + c1) (c1 = alpha |r|), and n counts the positive ratings.  Nonneg:
// NNLSSolver.solve in place of the Cholesky tail - warp 0 runs NNLS.solve on the same system (nnls_warp, its
// vectors in the staging area the accumulation no longer needs); there is no singular system.
template <bool kBatch, bool kImplicit = false, bool kNonneg = false>
__global__ void __launch_bounds__(kSolveThreads) als_solve_kernel(Side sd, const float* __restrict__ srcF,
                                                                  float* __restrict__ dstF, int k, double reg,
                                                                  unsigned long long* __restrict__ err,
                                                                  unsigned long long half_step, Batch bt,
                                                                  Implicit im) {
  static_assert(!(kBatch && kImplicit), "the batched fit is explicit only");
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint8_t s_keep[kChunk];
  int m = 0, exclude = -1, pos = blockIdx.x;
  if (kBatch) {
    m = blockIdx.x % bt.M;
    pos = blockIdx.x / bt.M;
    const BatchModel md = bt.models[m];
    if (half_step >= (unsigned long long)md.half_steps) return;   // this model has finished
    k = md.k;
    reg = md.reg;
    exclude = md.exclude;
    srcF += bt.to_users ? md.movie_off : md.user_off;
    dstF += bt.to_users ? md.user_off : md.movie_off;
    err += m;
  }
  const int nA = k * (k + 1) / 2;
  double* P = reinterpret_cast<double*>(smem);          // [nA] packed upper ata, then [k] atb
  double* B = P + nA;
  double* s_y = B + k;                                  // [k] the solves' published values
  float* s_x = reinterpret_cast<float*>(s_y + k);       // [kChunk][k] staged source factors
  float* s_r = s_x + kChunk * k;                        // [kChunk]
  uint8_t* s_i = reinterpret_cast<uint8_t*>(s_r + kChunk);   // [nA] row of each packed element
  uint8_t* s_j = s_i + nA;                                   // [nA] its column
  __shared__ int s_bad;
  __shared__ int s_nz[kMaxRank];
  const int tid = threadIdx.x;
  const int ent = sd.order[pos];
  const int lo0 = sd.off[ent], hi = sd.off[ent + 1];
  int n_train = hi - lo0;
  for (int e = tid; e < nA; e += kSolveThreads) {
    int j = 0;
    while ((j + 1) * (j + 2) / 2 <= e) ++j;
    s_j[e] = (uint8_t)j;
    s_i[e] = (uint8_t)(e - j * (j + 1) / 2);
  }
  for (int e = tid; e < nA + k; e += kSolveThreads) P[e] = kImplicit && e < nA ? im.yty[e] : 0.0;   // merge(YtY)
  if (tid == 0) s_bad = 0;
  if (kBatch || kImplicit) n_train = 0;
  for (int lo = lo0; lo < hi; lo += kChunk) {
    const int cn = min(kChunk, hi - lo);
    __syncthreads();                                    // the previous chunk is consumed
    for (int t = tid; t < cn * k; t += kSolveThreads) {
      const int c = t / k;
      s_x[t] = srcF[(size_t)sd.src[lo + c] * k + (t - c * k)];
    }
    for (int t = tid; t < cn; t += kSolveThreads) {
      s_r[t] = sd.r[lo + t];
      if (kBatch) s_keep[t] = bt.fold[lo + t] != exclude;
    }
    __syncthreads();
    if (kBatch)
      for (int c = 0; c < cn; ++c) n_train += s_keep[c];
    if (kImplicit)
      for (int c = 0; c < cn; ++c) n_train += s_r[c] > 0.0f;   // numExplicits
    for (int e = tid; e < nA + k; e += kSolveThreads) {
      double a = P[e];
      if (kImplicit) {
        if (e < nA) {                                   // dspr(c1): ap(i,j) += x(i) * (c1 * x(j)); none when c1 == 0
          const int i = s_i[e], j = s_j[e];
          for (int c = 0; c < cn; ++c) {
            const double c1 = __dmul_rn(im.alpha, (double)fabsf(s_r[c]));
            const float xj = s_x[c * k + j];
            if (c1 != 0.0 && xj != 0.0f)
              a = __dadd_rn(a, __dmul_rn((double)s_x[c * k + i], __dmul_rn(c1, (double)xj)));
          }
        } else {                                        // daxpy(1 + c1): atb(i) += (1 + c1) * x(i), for rating > 0
          const int i = e - nA;
          for (int c = 0; c < cn; ++c) {
            const float rv = s_r[c];
            if (rv > 0.0f) {
              const double b = __dadd_rn(1.0, __dmul_rn(im.alpha, (double)rv));
              a = __dadd_rn(a, __dmul_rn(b, (double)s_x[c * k + i]));
            }
          }
        }
      } else if (e < nA) {                              // dspr: ap(i,j) += x(i) * (1.0 * x(j)), skipped for x(j) == 0
        const int i = s_i[e], j = s_j[e];
        for (int c = 0; c < cn; ++c) {
          if (kBatch && !s_keep[c]) continue;
          const float xj = s_x[c * k + j];
          if (xj != 0.0f) a = __dadd_rn(a, __dmul_rn((double)s_x[c * k + i], (double)xj));
        }
      } else {                                          // daxpy: atb(i) += rating * x(i), skipped for rating == 0
        const int i = e - nA;
        for (int c = 0; c < cn; ++c) {
          if (kBatch && !s_keep[c]) continue;
          const float rv = s_r[c];
          if (rv != 0.0f) a = __dadd_rn(a, __dmul_rn((double)rv, (double)s_x[c * k + i]));
        }
      }
      P[e] = a;
    }
  }
  __syncthreads();
  if (kBatch) {
    if (tid == 0) bt.count[(size_t)m * sd.nE + ent] = n_train;
    if (n_train == 0) return;                           // not in this model (every thread has the same count)
  }
  const double lambda = __dmul_rn((double)n_train, reg);
  if (tid < k) P[tid * (tid + 1) / 2 + tid] = __dadd_rn(P[tid * (tid + 1) / 2 + tid], lambda);
  __syncthreads();
  if (kNonneg) {                                        // fillAtA's matrix is P read symmetrically
    if (tid < 32) nnls_warp(P, B, reinterpret_cast<double*>(s_x), k, dstF + (size_t)ent * k);
    return;
  }
  // dpptrf "U": in step r, U(r,r) = sqrt(a(r,r) - ddot(U(0:r,r), U(0:r,r))), then for c > r
  // U(r,c) = (a(r,c) - U(0,r) U(0,c) - ... - U(r-1,r) U(r-1,c)) / U(r,r): dtpsv's element, subtracted in order
  const int c = tid;
  const int bc = c * (c + 1) / 2;
  for (int r = 0; r < k; ++r) {
    const int br = r * (r + 1) / 2;
    if (c == r) {
      double dd = 0.0;
      for (int i = 0; i < r; ++i) dd = __dadd_rn(dd, __dmul_rn(P[br + i], P[br + i]));
      const double ajj = __dsub_rn(P[br + r], dd);
      if (!(ajj > 0.0)) s_bad = 1;                      // a non-positive or NaN pivot
      else P[br + r] = __dsqrt_rn(ajj);
    }
    __syncthreads();
    if (s_bad) {
      if (tid == 0) atomicMin(err, (half_step << 32) | (unsigned long long)ent);
      return;
    }
    if (c > r && c < k) {
      double t = P[bc + r];
      for (int i = 0; i < r; ++i) t = __dsub_rn(t, __dmul_rn(P[br + i], P[bc + i]));
      P[bc + r] = __ddiv_rn(t, P[br + r]);
    }
    __syncthreads();
  }
  // dtpsv "U", "T": y(j) = (b(j) - U(0,j) y(0) - ... - U(j-1,j) y(j-1)) / U(j,j); thread j keeps its running value
  double x = c < k ? B[c] : 0.0;
  for (int i = 0; i < k; ++i) {
    if (c == i) {
      x = __ddiv_rn(x, P[bc + c]);
      s_y[i] = x;
    }
    __syncthreads();
    if (c > i && c < k) x = __dsub_rn(x, __dmul_rn(P[bc + i], s_y[i]));
  }
  __syncthreads();
  // dtpsv "U", "N": for j = k-1 .. 0, if x(j) != 0: x(j) /= U(j,j), then x(i) -= x(j) U(i,j) for i < j
  for (int j = k - 1; j >= 0; --j) {
    if (c == j) {
      s_nz[j] = x != 0.0;
      if (x != 0.0) x = __ddiv_rn(x, P[bc + c]);
      s_y[j] = x;
    }
    __syncthreads();
    if (c < j && s_nz[j]) x = __dsub_rn(x, __dmul_rn(s_y[j], P[j * (j + 1) / 2 + c]));
  }
  if (c < k) dstF[(size_t)ent * k + c] = __double2float_rn(x);
}

// Spark's computeYtY: block b = blockIdx.y of the ten sums NormalEquation.add(y, 0.0) - dspr("U", k, 1.0, y, ap),
// skipped for y(j) == 0 - over its source entities members[boff[b] .. boff[b + 1]) (ascending id), from zero in
// double; thread blockIdx.x * kYtyThreads + threadIdx.x owns one packed element.  part [10][nA].
__global__ void __launch_bounds__(kYtyThreads) als_yty_kernel(const float* __restrict__ srcF, int k,
                                                              const int32_t* __restrict__ members,
                                                              const int32_t* __restrict__ boff,
                                                              double* __restrict__ part) {
  __shared__ float s_x[kChunk * kMaxRank];
  const int nA = k * (k + 1) / 2, b = blockIdx.y, tid = threadIdx.x;
  const int e = blockIdx.x * kYtyThreads + tid;
  int i = 0, j = 0;
  if (e < nA) {
    while ((j + 1) * (j + 2) / 2 <= e) ++j;
    i = e - j * (j + 1) / 2;
  }
  double a = 0.0;
  const int hi = boff[b + 1];
  for (int lo = boff[b]; lo < hi; lo += kChunk) {
    const int cn = min(kChunk, hi - lo);
    __syncthreads();                                    // the previous chunk is consumed
    for (int t = tid; t < cn * k; t += kYtyThreads) {
      const int c = t / k;
      s_x[t] = srcF[(size_t)members[lo + c] * k + (t - c * k)];
    }
    __syncthreads();
    if (e < nA)
      for (int c = 0; c < cn; ++c) {
        const float xj = s_x[c * k + j];
        if (xj != 0.0f) a = __dadd_rn(a, __dmul_rn((double)s_x[c * k + i], (double)xj));
      }
  }
  if (e < nA) part[(size_t)b * nA + e] = a;
}

// YtY = ((0 + B0) + B1) + ... + B9: NormalEquation.merge's daxpy(1.0) in block order
__global__ void als_yty_merge_kernel(const double* __restrict__ part, int nA, double* __restrict__ yty) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nA; e += gridDim.x * blockDim.x) {
    double y = 0.0;
    for (int b = 0; b < kYtyBlocks; ++b) y = __dadd_rn(y, part[(size_t)b * nA + e]);
    yty[e] = y;
  }
}

size_t solve_smem(int k) {
  const int nA = k * (k + 1) / 2;
  return sizeof(double) * (nA + 2 * k) + sizeof(float) * (kChunk * k + kChunk) + 2 * nA;
}

// candidate a ranks before b: higher score (NaN as -inf), then lower destination position
__device__ __forceinline__ bool rec_better(float sa, int ia, float sb, int ib) {
  const float ka = sa != sa ? -INFINITY : sa, kb = sb != sb ? -INFINITY : sb;
  return ka > kb || (ka == kb && ia < ib);
}

__global__ void __launch_bounds__(kRecWarps * 32) als_recommend_kernel(const float* __restrict__ src, int n_src,
                                                                       const int32_t* __restrict__ dst_ids,
                                                                       const float* __restrict__ dst, int n_dst,
                                                                       int k, int L, int32_t* __restrict__ out_ids,
                                                                       float* __restrict__ out_scores) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* s_dst = reinterpret_cast<float*>(smem);        // [k][kTile]
  float4* s_src = reinterpret_cast<float4*>(s_dst + k * kTile);   // [k][kRecWarps] 4 sources of a warp
  float* s_score = reinterpret_cast<float*>(s_src + k * kRecWarps);   // [kSrcPerBlock][L]
  int* s_pos = reinterpret_cast<int*>(s_score + kSrcPerBlock * L);
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int s0 = blockIdx.x * kSrcPerBlock;
  float* srcw = reinterpret_cast<float*>(s_src);
  for (int e = tid; e < kSrcPerBlock * k; e += blockDim.x) {   // source q's factor d at [d][q]
    const int q = e / k, d = e - q * k;
    srcw[d * kSrcPerBlock + q] = s0 + q < n_src ? src[(size_t)(s0 + q) * k + d] : 0.0f;
  }
  int cnt[kSrcPerWarp];
#pragma unroll
  for (int q = 0; q < kSrcPerWarp; ++q) cnt[q] = 0;
  for (int t0 = 0; t0 < n_dst; t0 += kTile) {
    const int tn = min(kTile, n_dst - t0);
    __syncthreads();
    for (int e = tid; e < tn * k; e += blockDim.x) {
      const int j = e / k, d = e - j * k;
      s_dst[d * kTile + j] = dst[(size_t)(t0 + j) * k + d];
    }
    __syncthreads();
    float acc[kSrcPerWarp][4];
#pragma unroll
    for (int q = 0; q < kSrcPerWarp; ++q)
#pragma unroll
      for (int t = 0; t < 4; ++t) acc[q][t] = 0.0f;
    for (int d = 0; d < k; ++d) {                       // dot += a(d) * b(d), in order from d = 0
      const float4 sv = s_src[d * kRecWarps + w];
      const float sq[4] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float x = s_dst[d * kTile + lane + 32 * t];
#pragma unroll
        for (int q = 0; q < kSrcPerWarp; ++q) acc[q][t] = __fadd_rn(acc[q][t], __fmul_rn(sq[q], x));
      }
    }
#pragma unroll
    for (int q = 0; q < kSrcPerWarp; ++q) {
      float* sc = s_score + (w * kSrcPerWarp + q) * L;
      int* ps = s_pos + (w * kSrcPerWarp + q) * L;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int jj = lane + 32 * t;
        const int pos = t0 + jj;
        const bool in = jj < tn && (cnt[q] < L || rec_better(acc[q][t], pos, sc[L - 1], ps[L - 1]));
        unsigned m = __ballot_sync(kFull, in);
        while (m) {
          const int from = __ffs(m) - 1;
          m &= m - 1;
          const float cs = __shfl_sync(kFull, acc[q][t], from);
          const int cp = __shfl_sync(kFull, pos, from);
          if (cnt[q] == L && !rec_better(cs, cp, sc[L - 1], ps[L - 1])) continue;   // the list moved on
          int at = 0;
          for (int b = 0; b < cnt[q]; b += 32) {
            const int e = b + lane;
            at += __popc(__ballot_sync(kFull, e < cnt[q] && rec_better(sc[e], ps[e], cs, cp)));
          }
          const int nc = min(cnt[q] + 1, L);
          float mv_s[kMaxNum / 32];
          int mv_p[kMaxNum / 32];
#pragma unroll
          for (int u = 0; u < kMaxNum / 32; ++u) {
            const int e = lane + 32 * u;
            if (e >= at && e + 1 < nc) { mv_s[u] = sc[e]; mv_p[u] = ps[e]; }
          }
          __syncwarp();
#pragma unroll
          for (int u = 0; u < kMaxNum / 32; ++u) {
            const int e = lane + 32 * u;
            if (e >= at && e + 1 < nc) { sc[e + 1] = mv_s[u]; ps[e + 1] = mv_p[u]; }
          }
          if (lane == 0) { sc[at] = cs; ps[at] = cp; }
          __syncwarp();
          cnt[q] = nc;
        }
      }
    }
  }
#pragma unroll
  for (int q = 0; q < kSrcPerWarp; ++q) {
    const int s = s0 + w * kSrcPerWarp + q;
    if (s >= n_src) continue;
    const float* sc = s_score + (w * kSrcPerWarp + q) * L;
    const int* ps = s_pos + (w * kSrcPerWarp + q) * L;
    for (int e = lane; e < L; e += 32) {
      out_ids[(size_t)s * L + e] = dst_ids[ps[e]];
      out_scores[(size_t)s * L + e] = sc[e];
    }
  }
}

// RankingMetrics per query, one warp per query: q's labels lab[off[q] .. off[q + 1]) sorted ascending (a set:
// equal neighbours count once), its predictions pred [q][L] best first.  Lane t looks up position base + t by
// binary search; lane 0 then walks the positions in order, summing in double with Spark's expressions: hits in the
// first min(L, k) over k, dcg and maxDcg over min(max(L, |lab|), k) positions with gain[i] = 1 / ln(i + 2), and
// the sum of (hits so far) / (i + 1) over every hit, over |lab|.  An empty label set scores 0.  out [3][n].
__global__ void __launch_bounds__(kRankWarps * 32) ranking_metrics_kernel(const int32_t* __restrict__ pred, int n,
                                                                          int L, const int32_t* __restrict__ off,
                                                                          const int32_t* __restrict__ lab, int k,
                                                                          const double* __restrict__ gain,
                                                                          double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  for (int q = blockIdx.x * kRankWarps + (threadIdx.x >> 5); q < n; q += gridDim.x * kRankWarps) {
    const int lo = off[q], hi = off[q + 1];
    int distinct = 0;
    for (int j = lo + lane; j < hi; j += 32) distinct += j == lo || lab[j] != lab[j - 1];
    distinct = __reduce_add_sync(kFull, distinct);
    if (distinct == 0) {
      if (lane == 0) out[q] = out[n + q] = out[2 * n + q] = 0.0;
      continue;
    }
    const int n_prec = min(L, k), n_ndcg = min(max(L, distinct), k), steps = max(L, n_ndcg);
    int cnt = 0, cnt_k = 0;
    double prec_sum = 0.0, dcg = 0.0, max_dcg = 0.0;
    for (int base = 0; base < steps; base += 32) {
      const int i = base + lane;
      bool hit = false;
      if (i < L) {
        const int32_t x = pred[(size_t)q * L + i];
        int a = lo, b = hi;                             // the first label >= x
        while (a < b) {
          const int m = (a + b) >> 1;
          if (lab[m] < x) a = m + 1;
          else b = m;
        }
        hit = a < hi && lab[a] == x;
      }
      const unsigned hits = __ballot_sync(kFull, hit);
      if (lane == 0)
        for (int t = 0; t < 32 && base + t < steps; ++t) {
          const int p = base + t;
          const bool h = (hits >> t) & 1u;
          if (h) {
            ++cnt;
            if (p < n_prec) ++cnt_k;
            prec_sum = __dadd_rn(prec_sum, __ddiv_rn((double)cnt, (double)(p + 1)));
          }
          if (p < n_ndcg) {
            if (h) dcg = __dadd_rn(dcg, gain[p]);
            if (p < distinct) max_dcg = __dadd_rn(max_dcg, gain[p]);
          }
        }
    }
    if (lane == 0) {
      out[q] = __ddiv_rn((double)cnt_k, (double)k);
      out[n + q] = __ddiv_rn(dcg, max_dcg);
      out[2 * n + q] = __ddiv_rn(prec_sum, (double)distinct);
    }
  }
}

int bits_for(int n) {
  int b = 1;
  while (b < 31 && (1 << b) < n) ++b;
  return b;
}

int check_params(int32_t rank, int32_t max_iter, double reg_param) {
  if (rank < 1 || rank > kMaxRank) return failf(SRS_ERR_INVALID, "rank %d outside 1..%d", rank, kMaxRank);
  if (max_iter < 1) return failf(SRS_ERR_INVALID, "max_iter %d is not positive", max_iter);
  if (!std::isfinite(reg_param) || reg_param < 0)
    return failf(SRS_ERR_INVALID, "reg_param %g is not finite and >= 0", reg_param);
  return SRS_OK;
}

int check_ratings(const int32_t* user_id, const int32_t* movie_id, const float* rating, int64_t n_ratings) {
  if (n_ratings < 1 || n_ratings > kMaxRatings)
    return failf(SRS_ERR_INVALID, "n_ratings %lld outside 1..%lld", (long long)n_ratings, (long long)kMaxRatings);
  if (!user_id || !movie_id || !rating) return failf(SRS_ERR_INVALID, "null ratings");
  for (int64_t i = 0; i < n_ratings; ++i) {
    if (user_id[i] < 0 || movie_id[i] < 0)
      return failf(SRS_ERR_INVALID, "rating %d: negative id (user %d, movie %d)", (int)i, user_id[i], movie_id[i]);
    if (!std::isfinite(rating[i])) return failf(SRS_ERR_INVALID, "rating %d is not finite", (int)i);
  }
  return SRS_OK;
}

// One rating set's dense ids and both layouts on the device (steps 1 and 2 of srs_als_fit_host)
struct Layouts {
  int nU = 0, nM = 0;
  int32_t *d_uids, *d_mids;            // the dense ids' raw ids, ascending
  int32_t *d_bm, *d_bu;                // input row of each by-movie / by-user layout position
  Side movies, users;
  std::vector<int32_t> uid;            // d_uids on the host
};

int build_layouts(HostCall& c, const int32_t* user_id, const int32_t* movie_id, const float* rating, int n,
                  int32_t user_capacity, int32_t movie_capacity, Layouts* L) {
  Scratch& sc = c.sc;
  cudaStream_t s = c.s;
  const int T = 256, G = grid_for(n, T);
  int32_t *d_user, *d_movie, *d_iota, *d_key, *d_perm_u, *d_perm_m, *d_head, *d_seg, *d_du, *d_dm;
  int32_t *d_uids, *d_ucnt, *d_mids, *d_mcnt, *d_bm, *d_bu, *d_src_m, *d_src_u;
  float *d_rating, *d_r_m, *d_r_u;
  int* d_count;
  CUDA_TRY(sc.alloc(&d_user, n)); CUDA_TRY(sc.alloc(&d_movie, n)); CUDA_TRY(sc.alloc(&d_rating, n));
  CUDA_TRY(sc.alloc(&d_iota, n)); CUDA_TRY(sc.alloc(&d_key, n)); CUDA_TRY(sc.alloc(&d_perm_u, n));
  CUDA_TRY(sc.alloc(&d_perm_m, n)); CUDA_TRY(sc.alloc(&d_head, n)); CUDA_TRY(sc.alloc(&d_seg, n));
  CUDA_TRY(sc.alloc(&d_du, n)); CUDA_TRY(sc.alloc(&d_dm, n)); CUDA_TRY(sc.alloc(&d_uids, n));
  CUDA_TRY(sc.alloc(&d_ucnt, n + 1)); CUDA_TRY(sc.alloc(&d_mids, n)); CUDA_TRY(sc.alloc(&d_mcnt, n + 1));
  CUDA_TRY(sc.alloc(&d_bm, n)); CUDA_TRY(sc.alloc(&d_bu, n)); CUDA_TRY(sc.alloc(&d_src_m, n));
  CUDA_TRY(sc.alloc(&d_src_u, n)); CUDA_TRY(sc.alloc(&d_r_m, n)); CUDA_TRY(sc.alloc(&d_r_u, n));
  CUDA_TRY(sc.alloc(&d_count, 2));
  CUDA_TRY(cudaMemcpyAsync(d_user, user_id, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_movie, movie_id, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_rating, rating, sizeof(float) * n, cudaMemcpyHostToDevice, s));
  als_iota_kernel<<<G, T, 0, s>>>(d_iota, n);
  LAUNCHED();

  // the dense ids: a stable sort by raw id, its run-length encoding, and each rating's segment
  const int32_t* raw[2] = {d_user, d_movie};
  int32_t* perm[2] = {d_perm_u, d_perm_m};
  int32_t* uniq[2] = {d_uids, d_mids};
  int32_t* cnt[2] = {d_ucnt, d_mcnt};
  int32_t* dense[2] = {d_du, d_dm};
  for (int side = 0; side < 2; ++side) {
    CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, raw[side], d_key, d_iota, perm[side], n, 0, 31, s));
    CUB_RUN(c, cub::DeviceRunLengthEncode::Encode(tmp__, tb__, d_key, uniq[side], cnt[side], d_count + side, n, s));
    als_head_kernel<<<G, T, 0, s>>>(d_key, n, d_head);
    LAUNCHED();
    CUB_RUN(c, cub::DeviceScan::InclusiveSum(tmp__, tb__, d_head, d_seg, n, s));
    als_scatter_kernel<<<G, T, 0, s>>>(perm[side], d_seg, n, dense[side]);
    LAUNCHED();
  }
  int counts[2];
  CUDA_TRY(cudaMemcpyAsync(counts, d_count, sizeof(counts), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  const int nU = counts[0], nM = counts[1];
  if (nU > user_capacity) return failf(SRS_ERR_RANGE, "%d users exceed capacity %d", nU, user_capacity);
  if (nM > movie_capacity) return failf(SRS_ERR_RANGE, "%d movies exceed capacity %d", nM, movie_capacity);
  L->uid.resize(nU);
  CUDA_TRY(cudaMemcpyAsync(L->uid.data(), d_uids, sizeof(int32_t) * nU, cudaMemcpyDeviceToHost, s));

  // by-movie layout: the (user, input)-ordered ratings stably sorted by dense movie; by-user: that by dense user
  als_key_kernel<<<G, T, 0, s>>>(d_perm_u, d_dm, n, d_key);
  LAUNCHED();
  CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_key, d_head, d_perm_u, d_bm, n, 0, bits_for(nM), s));
  als_key_kernel<<<G, T, 0, s>>>(d_bm, d_du, n, d_key);
  LAUNCHED();
  CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, d_key, d_head, d_bm, d_bu, n, 0, bits_for(nU), s));
  als_gather_kernel<<<G, T, 0, s>>>(d_bm, d_du, d_rating, n, d_src_m, d_r_m);
  LAUNCHED();
  als_gather_kernel<<<G, T, 0, s>>>(d_bu, d_dm, d_rating, n, d_src_u, d_r_u);
  LAUNCHED();
  // each side's offsets and its entities longest first (ties: lower index first)
  int32_t *d_moff, *d_uoff, *d_morder, *d_uorder;
  CUDA_TRY(sc.alloc(&d_moff, nM + 1)); CUDA_TRY(sc.alloc(&d_uoff, nU + 1));
  CUDA_TRY(sc.alloc(&d_morder, nM)); CUDA_TRY(sc.alloc(&d_uorder, nU));
  CUDA_TRY(cudaMemsetAsync(d_mcnt + nM, 0, sizeof(int32_t), s));
  CUDA_TRY(cudaMemsetAsync(d_ucnt + nU, 0, sizeof(int32_t), s));
  CUB_RUN(c, cub::DeviceScan::ExclusiveSum(tmp__, tb__, d_mcnt, d_moff, nM + 1, s));
  CUB_RUN(c, cub::DeviceScan::ExclusiveSum(tmp__, tb__, d_ucnt, d_uoff, nU + 1, s));
  CUB_RUN(c, cub::DeviceRadixSort::SortPairsDescending(tmp__, tb__, d_mcnt, d_key, d_iota, d_morder, nM, 0, 31, s));
  CUB_RUN(c, cub::DeviceRadixSort::SortPairsDescending(tmp__, tb__, d_ucnt, d_key, d_iota, d_uorder, nU, 0, 31, s));
  L->nU = nU;
  L->nM = nM;
  L->d_uids = d_uids;
  L->d_mids = d_mids;
  L->d_bm = d_bm;
  L->d_bu = d_bu;
  L->movies = Side{d_moff, d_src_m, d_r_m, d_morder, nM};
  L->users = Side{d_uoff, d_src_u, d_r_u, d_uorder, nU};
  return SRS_OK;
}

// srs_als_fit_host, srs_als_fit_implicit_host and srs_als_fit_nonnegative_host: every check, then the fit.
// `alpha` null: explicit feedback; `nonneg`: NNLSSolver in place of CholeskySolver.
int fit_single(const int32_t* user_id, const int32_t* movie_id, const float* rating, int64_t n_ratings,
               const srs_als_params* params, const double* alpha, bool nonneg, int32_t device, int32_t user_capacity,
               int32_t movie_capacity, int32_t* user_ids, float* user_factors, int32_t* n_users, int32_t* movie_ids,
               float* movie_factors, int32_t* n_movies) {
  if (!n_users || !n_movies) return failf(SRS_ERR_INVALID, "null n_users or n_movies");
  *n_users = 0;
  *n_movies = 0;
  if (!params) return failf(SRS_ERR_INVALID, "null params");
  const srs_als_params hp = *params;
  PROPAGATE(check_params(hp.rank, hp.max_iter, hp.reg_param));
  if (alpha && (!std::isfinite(*alpha) || *alpha < 0))
    return failf(SRS_ERR_INVALID, "alpha %g is not finite and >= 0", *alpha);
  PROPAGATE(check_ratings(user_id, movie_id, rating, n_ratings));
  if (user_capacity < 0 || movie_capacity < 0 || (user_capacity > 0 && (!user_ids || !user_factors)) ||
      (movie_capacity > 0 && (!movie_ids || !movie_factors)))
    return failf(SRS_ERR_INVALID, "negative capacity or null outputs");

  HostCall c;
  PROPAGATE(c.begin(device));
  Scratch& sc = c.sc;
  cudaStream_t s = c.s;
  const int k = hp.rank;
  Layouts L;
  PROPAGATE(build_layouts(c, user_id, movie_id, rating, (int)n_ratings, user_capacity, movie_capacity, &L));
  const int nU = L.nU, nM = L.nM;

  // the users' initial factors, drawn on the host
  std::vector<float> init((size_t)nU * k);
  for (int u = 0; u < nU; ++u) init_factor(hp.seed, L.uid[u], k, init.data() + (size_t)u * k);
  float *d_uf, *d_mf;
  unsigned long long* d_err;
  CUDA_TRY(sc.alloc(&d_uf, (size_t)nU * k)); CUDA_TRY(sc.alloc(&d_mf, (size_t)nM * k)); CUDA_TRY(sc.alloc(&d_err, 1));
  CUDA_TRY(cudaMemcpyAsync(d_uf, init.data(), sizeof(float) * init.size(), cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemsetAsync(d_err, 0xff, sizeof(unsigned long long), s));
  const size_t sm = solve_smem(k);
  if (!alpha) {
    auto* solve = nonneg ? als_solve_kernel<false, false, true> : als_solve_kernel<false>;
    for (int it = 0; it < hp.max_iter; ++it) {
      solve<<<nM, kSolveThreads, sm, s>>>(L.movies, d_uf, d_mf, k, hp.reg_param, d_err, 2ull * it, Batch{},
                                          Implicit{});
      LAUNCHED();
      solve<<<nU, kSolveThreads, sm, s>>>(L.users, d_mf, d_uf, k, hp.reg_param, d_err, 2ull * it + 1, Batch{},
                                          Implicit{});
      LAUNCHED();
    }
  } else {
    // YtY's blocks: each side's dense entities grouped by raw id mod 10, ascending id within a block
    std::vector<int32_t> mid(nM);
    CUDA_TRY(cudaMemcpyAsync(mid.data(), L.d_mids, sizeof(int32_t) * nM, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    int32_t *d_umem, *d_mmem, *d_uboff, *d_mboff;
    const std::vector<int32_t>* ids[2] = {&L.uid, &mid};
    int32_t** mem[2] = {&d_umem, &d_mmem};
    int32_t** boff[2] = {&d_uboff, &d_mboff};
    for (int side = 0; side < 2; ++side) {
      const std::vector<int32_t>& id = *ids[side];
      std::vector<int32_t> members, off(kYtyBlocks + 1, 0);
      members.reserve(id.size());
      for (int b = 0; b < kYtyBlocks; ++b) {
        for (size_t e = 0; e < id.size(); ++e)
          if (id[e] % kYtyBlocks == b) members.push_back((int32_t)e);
        off[b + 1] = (int32_t)members.size();
      }
      PROPAGATE(c.upload(mem[side], members.data(), members.size()));
      PROPAGATE(c.upload(boff[side], off.data(), off.size()));
    }
    const int nA = k * (k + 1) / 2;
    double *d_part, *d_yty;
    CUDA_TRY(sc.alloc(&d_part, (size_t)kYtyBlocks * nA)); CUDA_TRY(sc.alloc(&d_yty, nA));
    const dim3 yg((nA + kYtyThreads - 1) / kYtyThreads, kYtyBlocks);
    const Implicit im{d_yty, *alpha};
    auto* solve = nonneg ? als_solve_kernel<false, true, true> : als_solve_kernel<false, true>;
    for (int it = 0; it < hp.max_iter; ++it)
      for (int half = 0; half < 2; ++half) {            // the movies from the users, then the users from the movies
        const bool to_users = half == 1;
        const float* src = to_users ? d_mf : d_uf;
        als_yty_kernel<<<yg, kYtyThreads, 0, s>>>(src, k, to_users ? d_mmem : d_umem, to_users ? d_mboff : d_uboff,
                                                  d_part);
        LAUNCHED();
        als_yty_merge_kernel<<<grid_for(nA, 256), 256, 0, s>>>(d_part, nA, d_yty);
        LAUNCHED();
        solve<<<to_users ? nU : nM, kSolveThreads, sm, s>>>(to_users ? L.users : L.movies, src,
                                                            to_users ? d_uf : d_mf, k, hp.reg_param, d_err,
                                                            2ull * it + half, Batch{}, im);
        LAUNCHED();
      }
  }
  unsigned long long err = 0;
  CUDA_TRY(cudaMemcpyAsync(&err, d_err, sizeof(err), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  if (err != ~0ull) {
    const int hs = (int)(err >> 32), ent = (int)(err & 0xffffffffu);
    int32_t id = 0;
    CUDA_TRY(cudaMemcpy(&id, (hs & 1 ? L.d_uids : L.d_mids) + ent, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return failf(SRS_ERR_INVALID, "singular normal equations for %s %d in iteration %d (a pivot <= 0 or NaN)",
                    hs & 1 ? "user" : "movie", id, hs / 2 + 1);
  }
  CUDA_TRY(cudaMemcpyAsync(user_ids, L.d_uids, sizeof(int32_t) * nU, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(user_factors, d_uf, sizeof(float) * nU * k, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(movie_ids, L.d_mids, sizeof(int32_t) * nM, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(movie_factors, d_mf, sizeof(float) * nM * k, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  *n_users = nU;
  *n_movies = nM;
  return SRS_OK;
}

}  // namespace
}  // namespace srs

extern "C" int srs_als_fit_host(const int32_t* user_id, const int32_t* movie_id, const float* rating,
                                int64_t n_ratings, const srs_als_params* params, int32_t device,
                                int32_t user_capacity, int32_t movie_capacity, int32_t* user_ids,
                                float* user_factors, int32_t* n_users, int32_t* movie_ids, float* movie_factors,
                                int32_t* n_movies) {
  return srs::fit_single(user_id, movie_id, rating, n_ratings, params, nullptr, false, device, user_capacity,
                         movie_capacity, user_ids, user_factors, n_users, movie_ids, movie_factors, n_movies);
}

extern "C" int srs_als_fit_implicit_host(const int32_t* user_id, const int32_t* movie_id, const float* rating,
                                         int64_t n_ratings, const srs_als_params* params, int32_t device,
                                         int32_t user_capacity, int32_t movie_capacity, int32_t* user_ids,
                                         float* user_factors, int32_t* n_users, int32_t* movie_ids,
                                         float* movie_factors, int32_t* n_movies, double alpha) {
  return srs::fit_single(user_id, movie_id, rating, n_ratings, params, &alpha, false, device, user_capacity,
                         movie_capacity, user_ids, user_factors, n_users, movie_ids, movie_factors, n_movies);
}

extern "C" int srs_als_fit_nonnegative_host(const int32_t* user_id, const int32_t* movie_id, const float* rating,
                                            int64_t n_ratings, const srs_als_params* params, int32_t device,
                                            int32_t user_capacity, int32_t movie_capacity, int32_t* user_ids,
                                            float* user_factors, int32_t* n_users, int32_t* movie_ids,
                                            float* movie_factors, int32_t* n_movies, int32_t implicit_prefs,
                                            double alpha) {
  if (implicit_prefs != 0 && implicit_prefs != 1) {
    if (n_users) *n_users = 0;
    if (n_movies) *n_movies = 0;
    return srs::failf(SRS_ERR_INVALID, "implicit_prefs %d is not 0 or 1", implicit_prefs);
  }
  return srs::fit_single(user_id, movie_id, rating, n_ratings, params, implicit_prefs ? &alpha : nullptr, true,
                         device, user_capacity, movie_capacity, user_ids, user_factors, n_users, movie_ids,
                         movie_factors, n_movies);
}

using namespace srs;

namespace {

// srs_als_fit_folds_host and srs_als_fit_folds_nonnegative_host: every check, then the batched fit.  `nonneg`
// [n_models] (null: none) picks each model's solver; the NNLS models run in a launch of their own per half-step,
// over their own slice of the model list.
int fit_folds(const int32_t* user_id, const int32_t* movie_id, const float* rating, const int32_t* fold,
              int64_t n_ratings, int32_t n_folds, const srs_als_model* models, const int32_t* nonneg,
              int32_t n_models, uint64_t seed, int32_t device, int32_t user_capacity, int32_t movie_capacity,
              int32_t* user_ids, float* user_factors, int32_t* n_users, int32_t* movie_ids, float* movie_factors,
              int32_t* n_movies) {
  if (n_models < 1 || n_models > kMaxModels)
    return failf(SRS_ERR_INVALID, "n_models %d outside 1..%d", n_models, kMaxModels);
  if (!models || !n_users || !n_movies) return failf(SRS_ERR_INVALID, "null models, n_users or n_movies");
  for (int m = 0; m < n_models; ++m) n_users[m] = n_movies[m] = 0;
  if (n_folds < 2 || n_folds > kMaxFolds)
    return failf(SRS_ERR_INVALID, "n_folds %d outside 2..%d", n_folds, kMaxFolds);
  const std::vector<srs_als_model> md(models, models + n_models);
  for (int m = 0; m < n_models; ++m) {
    if (int rc = check_params(md[m].rank, md[m].max_iter, md[m].reg_param))
      return failf(rc, "model %d: %s", m, srs_last_error());
    if (md[m].exclude_fold < -1 || md[m].exclude_fold >= n_folds)
      return failf(SRS_ERR_INVALID, "model %d: exclude_fold %d outside -1..%d", m, md[m].exclude_fold, n_folds - 1);
    if (nonneg && nonneg[m] != 0 && nonneg[m] != 1)
      return failf(SRS_ERR_INVALID, "model %d: nonnegative %d is not 0 or 1", m, nonneg[m]);
  }
  PROPAGATE(check_ratings(user_id, movie_id, rating, n_ratings));
  if (!fold) return failf(SRS_ERR_INVALID, "null fold");
  if (user_capacity < 0 || movie_capacity < 0 || (user_capacity > 0 && (!user_ids || !user_factors)) ||
      (movie_capacity > 0 && (!movie_ids || !movie_factors)))
    return failf(SRS_ERR_INVALID, "negative capacity or null outputs");
  const int n = (int)n_ratings;
  std::vector<int64_t> in_fold(n_folds, 0);
  for (int i = 0; i < n; ++i) {
    if (fold[i] < 0 || fold[i] >= n_folds)
      return failf(SRS_ERR_INVALID, "rating %d: fold %d outside 0..%d", i, fold[i], n_folds - 1);
    ++in_fold[fold[i]];
  }
  for (int m = 0; m < n_models; ++m)
    if (md[m].exclude_fold >= 0 && in_fold[md[m].exclude_fold] == n)
      return failf(SRS_ERR_INVALID, "model %d: no training ratings (every rating is in fold %d)", m,
                      md[m].exclude_fold);

  HostCall c;
  PROPAGATE(c.begin(device));
  Scratch& sc = c.sc;
  cudaStream_t s = c.s;
  Layouts L;
  PROPAGATE(build_layouts(c, user_id, movie_id, rating, n, user_capacity, movie_capacity, &L));
  const int nU = L.nU, nM = L.nM, M = n_models, T = 256, G = grid_for(n, T);

  // each model's factors over every dense id of the whole set; the initial user factors depend on the rank only
  std::vector<BatchModel> bm(M);
  size_t uf_total = 0, mf_total = 0;
  int kmax = 1, half_steps = 0;
  for (int m = 0; m < M; ++m) {
    bm[m] = BatchModel{md[m].rank, 2 * md[m].max_iter, md[m].reg_param, md[m].exclude_fold, uf_total, mf_total};
    uf_total += (size_t)nU * md[m].rank;
    mf_total += (size_t)nM * md[m].rank;
    kmax = std::max(kmax, md[m].rank);
    half_steps = std::max(half_steps, 2 * md[m].max_iter);
  }
  // slot[m]: model m's place in the device list - the Cholesky models first, then the M_nn NNLS models
  std::vector<int> slot(M);
  int M_nn = 0;
  for (int m = 0; m < M; ++m) M_nn += nonneg && nonneg[m];
  for (int m = 0, a = 0, b = M - M_nn; m < M; ++m) slot[m] = nonneg && nonneg[m] ? b++ : a++;
  std::vector<BatchModel> dev_bm(M);
  for (int m = 0; m < M; ++m) dev_bm[slot[m]] = bm[m];
  std::vector<float> init(uf_total);
  std::vector<int> drawn(kMaxRank + 1, -1);            // the first model of each rank
  for (int m = 0; m < M; ++m) {
    const int k = md[m].rank;
    float* dst = init.data() + bm[m].user_off;
    if (drawn[k] >= 0) {
      std::copy_n(init.data() + bm[drawn[k]].user_off, (size_t)nU * k, dst);
      continue;
    }
    drawn[k] = m;
    for (int u = 0; u < nU; ++u) init_factor(seed, L.uid[u], k, dst + (size_t)u * k);
  }
  int32_t *d_fold, *d_fold_m, *d_fold_u, *d_cnt_m, *d_cnt_u;
  float *d_uf, *d_mf;
  BatchModel* d_models;
  unsigned long long* d_err;
  CUDA_TRY(sc.alloc(&d_fold, n)); CUDA_TRY(sc.alloc(&d_fold_m, n)); CUDA_TRY(sc.alloc(&d_fold_u, n));
  CUDA_TRY(sc.alloc(&d_cnt_m, (size_t)M * nM)); CUDA_TRY(sc.alloc(&d_cnt_u, (size_t)M * nU));
  CUDA_TRY(sc.alloc(&d_uf, uf_total)); CUDA_TRY(sc.alloc(&d_mf, mf_total));
  CUDA_TRY(sc.alloc(&d_models, M)); CUDA_TRY(sc.alloc(&d_err, M));
  CUDA_TRY(cudaMemcpyAsync(d_fold, fold, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_uf, init.data(), sizeof(float) * uf_total, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_models, dev_bm.data(), sizeof(BatchModel) * M, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemsetAsync(d_err, 0xff, sizeof(unsigned long long) * M, s));
  als_key_kernel<<<G, T, 0, s>>>(L.d_bm, d_fold, n, d_fold_m);      // each layout's fold ids
  LAUNCHED();
  als_key_kernel<<<G, T, 0, s>>>(L.d_bu, d_fold, n, d_fold_u);
  LAUNCHED();
  // one launch per half-step for every Cholesky model and one for every NNLS model: a model past its max_iter
  // exits at once
  const size_t sm = solve_smem(kmax);
  const int M_ch = M - M_nn;
  for (int h = 0; h < half_steps; ++h) {
    const bool to_users = h & 1;
    const int nE = to_users ? nU : nM;
    int32_t* cnt = to_users ? d_cnt_u : d_cnt_m;
    const int32_t* fd = to_users ? d_fold_u : d_fold_m;
    if (M_ch > 0) {
      als_solve_kernel<true><<<(unsigned)((int64_t)nE * M_ch), kSolveThreads, sm, s>>>(
          to_users ? L.users : L.movies, to_users ? d_mf : d_uf, to_users ? d_uf : d_mf, 0, 0.0, d_err,
          (unsigned long long)h, Batch{d_models, fd, cnt, M_ch, to_users}, Implicit{});
      LAUNCHED();
    }
    if (M_nn > 0) {
      als_solve_kernel<true, false, true><<<(unsigned)((int64_t)nE * M_nn), kSolveThreads, sm, s>>>(
          to_users ? L.users : L.movies, to_users ? d_mf : d_uf, to_users ? d_uf : d_mf, 0, 0.0, d_err + M_ch,
          (unsigned long long)h, Batch{d_models + M_ch, fd, cnt + (size_t)M_ch * nE, M_nn, to_users}, Implicit{});
      LAUNCHED();
    }
  }
  std::vector<unsigned long long> err(M);
  CUDA_TRY(cudaMemcpyAsync(err.data(), d_err, sizeof(unsigned long long) * M, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (int m = 0; m < M; ++m) {
    const unsigned long long e = err[slot[m]];
    if (e == ~0ull) continue;
    const int hs = (int)(e >> 32), ent = (int)(e & 0xffffffffu);
    int32_t id = 0;
    CUDA_TRY(cudaMemcpy(&id, (hs & 1 ? L.d_uids : L.d_mids) + ent, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return failf(SRS_ERR_INVALID,
                    "model %d: singular normal equations for %s %d in iteration %d (a pivot <= 0 or NaN)", m,
                    hs & 1 ? "user" : "movie", id, hs / 2 + 1);
  }
  std::vector<int32_t> mid(nM), cnt_u((size_t)M * nU), cnt_m((size_t)M * nM);
  std::vector<float> uf(uf_total), mf(mf_total);
  CUDA_TRY(cudaMemcpyAsync(mid.data(), L.d_mids, sizeof(int32_t) * nM, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(cnt_u.data(), d_cnt_u, sizeof(int32_t) * cnt_u.size(), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(cnt_m.data(), d_cnt_m, sizeof(int32_t) * cnt_m.size(), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(uf.data(), d_uf, sizeof(float) * uf_total, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(mf.data(), d_mf, sizeof(float) * mf_total, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  // model m's entities are those with a training rating in it, ascending; its outputs start after the models before
  size_t uo = 0, mo = 0;
  for (int m = 0; m < M; ++m) {
    const int k = md[m].rank;
    int32_t nu = 0, nm = 0;
    for (int u = 0; u < nU; ++u) {
      if (!cnt_u[(size_t)slot[m] * nU + u]) continue;
      user_ids[(size_t)m * user_capacity + nu] = L.uid[u];
      std::copy_n(uf.data() + bm[m].user_off + (size_t)u * k, k, user_factors + uo + (size_t)nu * k);
      ++nu;
    }
    for (int e = 0; e < nM; ++e) {
      if (!cnt_m[(size_t)slot[m] * nM + e]) continue;
      movie_ids[(size_t)m * movie_capacity + nm] = mid[e];
      std::copy_n(mf.data() + bm[m].movie_off + (size_t)e * k, k, movie_factors + mo + (size_t)nm * k);
      ++nm;
    }
    n_users[m] = nu;
    n_movies[m] = nm;
    uo += (size_t)user_capacity * k;
    mo += (size_t)movie_capacity * k;
  }
  return SRS_OK;
}

}  // namespace

extern "C" int srs_als_fit_folds_host(const int32_t* user_id, const int32_t* movie_id, const float* rating,
                                      const int32_t* fold, int64_t n_ratings, int32_t n_folds,
                                      const srs_als_model* models, int32_t n_models, uint64_t seed, int32_t device,
                                      int32_t user_capacity, int32_t movie_capacity, int32_t* user_ids,
                                      float* user_factors, int32_t* n_users, int32_t* movie_ids,
                                      float* movie_factors, int32_t* n_movies) {
  return fit_folds(user_id, movie_id, rating, fold, n_ratings, n_folds, models, nullptr, n_models, seed, device,
                   user_capacity, movie_capacity, user_ids, user_factors, n_users, movie_ids, movie_factors, n_movies);
}

extern "C" int srs_als_fit_folds_nonnegative_host(const int32_t* user_id, const int32_t* movie_id,
                                                  const float* rating, const int32_t* fold, int64_t n_ratings,
                                                  int32_t n_folds, const srs_als_model* models, int32_t n_models,
                                                  uint64_t seed, int32_t device, int32_t user_capacity,
                                                  int32_t movie_capacity, int32_t* user_ids, float* user_factors,
                                                  int32_t* n_users, int32_t* movie_ids, float* movie_factors,
                                                  int32_t* n_movies, const int32_t* nonnegative) {
  if (!nonnegative) {
    if (n_users && n_models >= 1 && n_models <= kMaxModels)
      for (int m = 0; m < n_models; ++m) n_users[m] = 0;
    if (n_movies && n_models >= 1 && n_models <= kMaxModels)
      for (int m = 0; m < n_models; ++m) n_movies[m] = 0;
    return failf(SRS_ERR_INVALID, "null nonnegative");
  }
  return fit_folds(user_id, movie_id, rating, fold, n_ratings, n_folds, models, nonnegative, n_models, seed, device,
                   user_capacity, movie_capacity, user_ids, user_factors, n_users, movie_ids, movie_factors, n_movies);
}

extern "C" int srs_als_recommend_host(const float* src_factors, int32_t n_src, const int32_t* dst_ids,
                                      const float* dst_factors, int32_t n_dst, int32_t rank, int32_t num,
                                      int32_t device, int32_t* out_ids, float* out_scores) {
  if (rank < 1 || rank > kMaxRank) return failf(SRS_ERR_INVALID, "rank %d outside 1..%d", rank, kMaxRank);
  if (num < 1 || num > kMaxNum) return failf(SRS_ERR_INVALID, "num %d outside 1..%d", num, kMaxNum);
  if (n_src < 0 || n_dst < 0) return failf(SRS_ERR_INVALID, "negative n_src or n_dst");
  if ((n_src && !src_factors) || (n_dst && (!dst_ids || !dst_factors)) ||
      (n_src && n_dst && (!out_ids || !out_scores)))
    return failf(SRS_ERR_INVALID, "null factors, ids or outputs");
  for (int32_t i = 1; i < n_dst; ++i)
    if (dst_ids[i] <= dst_ids[i - 1])
      return failf(SRS_ERR_INVALID, "destination ids are not strictly ascending at %d", i);
  for (int64_t i = 0; i < (int64_t)n_src * rank; ++i)
    if (!std::isfinite(src_factors[i])) return failf(SRS_ERR_INVALID, "source factor element %lld is not finite", (long long)i);
  for (int64_t i = 0; i < (int64_t)n_dst * rank; ++i)
    if (!std::isfinite(dst_factors[i]))
      return failf(SRS_ERR_INVALID, "destination factor element %lld is not finite", (long long)i);
  if (n_src == 0 || n_dst == 0) return SRS_OK;
  HostCall c;
  PROPAGATE(c.begin(device));
  Scratch& sc = c.sc;
  cudaStream_t s = c.s;
  const int L = std::min(num, n_dst), k = rank;
  float *d_src, *d_dst, *d_scores;
  int32_t *d_dids, *d_ids;
  CUDA_TRY(sc.alloc(&d_src, (size_t)n_src * k)); CUDA_TRY(sc.alloc(&d_dst, (size_t)n_dst * k));
  CUDA_TRY(sc.alloc(&d_dids, n_dst)); CUDA_TRY(sc.alloc(&d_ids, (size_t)n_src * L));
  CUDA_TRY(sc.alloc(&d_scores, (size_t)n_src * L));
  CUDA_TRY(cudaMemcpyAsync(d_src, src_factors, sizeof(float) * n_src * k, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_dst, dst_factors, sizeof(float) * n_dst * k, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_dids, dst_ids, sizeof(int32_t) * n_dst, cudaMemcpyHostToDevice, s));
  const size_t sm = sizeof(float) * k * kTile + sizeof(float4) * k * kRecWarps + (sizeof(float) + sizeof(int)) *
                    kSrcPerBlock * L;
  CUDA_TRY(cudaFuncSetAttribute(als_recommend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  als_recommend_kernel<<<(n_src + kSrcPerBlock - 1) / kSrcPerBlock, kRecWarps * 32, sm, s>>>(
      d_src, n_src, d_dids, d_dst, n_dst, k, L, d_ids, d_scores);
  LAUNCHED();
  CUDA_TRY(cudaMemcpyAsync(out_ids, d_ids, sizeof(int32_t) * n_src * L, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(out_scores, d_scores, sizeof(float) * n_src * L, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  return SRS_OK;
}

extern "C" int srs_ranking_metrics_host(const int32_t* pred_ids, int32_t n_queries, int32_t pred_len,
                                        const int32_t* label_off, const int32_t* label_ids, int32_t k,
                                        int32_t device, double* per_query, double* means) {
  if (!means) return failf(SRS_ERR_INVALID, "null means");
  if (n_queries < 0 || pred_len < 0) return failf(SRS_ERR_INVALID, "negative n_queries or pred_len");
  if (k < 1) return failf(SRS_ERR_INVALID, "k %d is not positive", k);
  if ((int64_t)n_queries * pred_len > INT32_MAX)
    return failf(SRS_ERR_INVALID, "%d x %d predictions exceed %d", n_queries, pred_len, INT32_MAX);
  if (n_queries > 0 && (!label_off || (pred_len > 0 && !pred_ids)))
    return failf(SRS_ERR_INVALID, "null predictions or label offsets");
  int32_t max_lab = 0;
  if (n_queries > 0) {
    if (label_off[0] != 0) return failf(SRS_ERR_INVALID, "label_off[0] is %d, not 0", label_off[0]);
    for (int32_t q = 0; q < n_queries; ++q) {
      if (label_off[q + 1] < label_off[q])
        return failf(SRS_ERR_INVALID, "label offsets decrease at query %d", q);
      max_lab = std::max(max_lab, label_off[q + 1] - label_off[q]);
    }
    if (label_off[n_queries] > 0 && !label_ids) return failf(SRS_ERR_INVALID, "null label ids");
  }
  if (n_queries == 0) {                               // no query: the means are undefined
    means[0] = means[1] = means[2] = NAN;
    return SRS_OK;
  }
  const int nnz = label_off[n_queries];
  // gain[i] = 1 / ln(i + 2) for every position an NDCG loop can reach, on the host (no device transcendental)
  const int n_gain = std::min(k, std::max(pred_len, max_lab));
  std::vector<double> gain(std::max(n_gain, 1), 0.0);
  for (int i = 0; i < n_gain; ++i) gain[i] = 1.0 / std::log((double)(i + 2));

  HostCall c;
  PROPAGATE(c.begin(device));
  cudaStream_t s = c.s;
  int32_t *d_pred, *d_off, *d_lab_in, *d_lab;
  double *d_gain, *d_out;
  PROPAGATE(c.upload(&d_pred, pred_ids, (size_t)n_queries * pred_len));
  PROPAGATE(c.upload(&d_off, label_off, (size_t)n_queries + 1));
  PROPAGATE(c.upload(&d_lab_in, label_ids, (size_t)nnz));
  PROPAGATE(c.upload(&d_gain, gain.data(), gain.size()));
  CUDA_TRY(c.sc.alloc(&d_lab, (size_t)nnz));
  CUDA_TRY(c.sc.alloc(&d_out, (size_t)3 * n_queries));
  if (nnz > 0)                                        // each query's labels ascending: a set by its runs
    CUB_RUN(c, cub::DeviceSegmentedRadixSort::SortKeys(tmp__, tb__, d_lab_in, d_lab, nnz, n_queries, d_off,
                                                       d_off + 1, 0, 32, s));
  const int blocks = (int)std::min<int64_t>(((int64_t)n_queries + kRankWarps - 1) / kRankWarps, kMaxGridBlocks);
  ranking_metrics_kernel<<<blocks, kRankWarps * 32, 0, s>>>(d_pred, n_queries, pred_len, d_off, d_lab, k, d_gain,
                                                           d_out);
  LAUNCHED();
  std::vector<double> v((size_t)3 * n_queries);
  CUDA_TRY(cudaMemcpyAsync(v.data(), d_out, sizeof(double) * v.size(), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (int m = 0; m < 3; ++m) {                       // StatCounter's mean, in query order: mu += (x - mu) / n
    double mu = 0.0;
    for (int32_t q = 0; q < n_queries; ++q) mu = mu + (v[(size_t)m * n_queries + q] - mu) / (double)(q + 1);
    means[m] = mu;
  }
  if (per_query) std::copy(v.begin(), v.end(), per_query);
  return SRS_OK;
}
