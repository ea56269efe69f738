// trainer.cu - `model.fit` on the device: the C ABI's srs_trainer (include/srs_ctr.h), which trains NeuralCF
// (neural_cf_model_1, NeuralCF.py:74-91; DESIGN.md section 4.8), DeepFM (DeepFM.py; section 4.9), Wide&Deep
// (WideNDeep.py; section 4.18), DeepFM_v2 (DeepFM_v2.py; section 4.19), DIEN (DIEN.py; section 4.20, its fit in
// srs_trainer_fit_dien_host) and two towers (neural_cf_model_2 with its final Dense, NeuralCF.py:57-70; section
// 4.27), and the kernels the models share: dedupe and the two forms of Adam.  Each model's step kernel is in its own
// file.  Two towers runs NeuralCF's column of the table below with twotowers_train_step_kernel as its step.
//
// A step of B rows (rows order[off .. off + B) of the uploaded dataset) is these launches in this order, with no
// host synchronisation; T is DIEN's hist_len:
//
// | launch                     | NeuralCF | DeepFM    | Wide&Deep     | DeepFM_v2 | DIEN                   |
// |----------------------------|----------|-----------|---------------|-----------|------------------------|
// | <model>_train_step_kernel  | ncf      | deepfm    | widendeep     | deepfm2   | dien                   |
// | table_grad_kernel, tables  | 2B       | 6B        | 10B           | 4B        | (2T + 3) B             |
// | table_grad_kernel, one-hot | -        | 4B        | B             | 4B        | -                      |
// | table_adam_kernel<false>   | 2 tables | 6 tables  | 10 tables     | 4 tables  | 4 tables               |
// | table_adam_kernel<true>    | -        | fm1_width | cross_buckets | fm1_width | -                      |
// | dense_adam_kernel          | 1        | 1         | 1             | 1         | 1                      |
// | dien_final_loss_kernel     | -        | -         | -             | -         | 1                      |
// | metrics_update_kernel      | 1        | 1         | 1             | 1         | 1, with its histogram  |
// | launches per step          | 5        | 7         | 7             | 7         | 6                      |
// | per epoch                  | -        | deepfm_   | widendeep_    | deepfm_   | launch_auc_value's 3   |
// |                            |          | permute   | permute       | permute   |                        |
//
// The step kernel computes the forward and backward, writes each row's table (and one-hot) entries with their
// gradients to lists and the Dense gradients as per-CTA partials summed over the CTA's rows in row order.
// table_grad_kernel dedupes each list (TF's _deduplicate_indexed_slices), table_adam_kernel applies Keras's sparse
// Adam to EVERY table row and ApplyAdam to every one-hot row, dense_adam_kernel sums the partials in CTA order, applies
// ApplyAdam to the Dense weights and advances the device-resident iteration counter.  The tile models read the
// epoch's rows permuted once per epoch; NeuralCF, two towers and DIEN read the dataset through the order.  No float
// atomics: every sum has a fixed order, so a fit is bitwise reproducible.
//
// Sample weights (srs_trainer_fit_weighted_host, srs_trainer_evaluate_weighted_host; DESIGN.md section 4.28) add no
// launch: the dataset's weight column is uploaded beside the labels, the step kernels scale dL/dz by it (NeuralCF and
// two towers read weight[order[i]] and pass the step's weights on, the permute kernels carry it for the tile
// models), and metrics_update_kernel's weighted instantiation replaces the unweighted one.
//
// Validation (srs_trainer_fit_validate_host) and srs_trainer_evaluate_host run the serving forward over the
// trainer's arrays (ncf_kernel, deepfm_kernel, embmlp_kernel, deepfm2_kernel) and one metrics_update_kernel over all
// the rows: two launches, with the bits of a CTRModel built from the exported weights.  The trainer's arrays hold the
// weights where the serving builders put them: both place them through placement.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"
#include "kernels.h"
#include "placement.h"

namespace srs {

namespace {

constexpr int kAdamThreads = 512;     // the one CTA of dense_adam_kernel

struct AdamHp { float lr, b1, b2, eps; };

// Keras's step size for t = iterations + 1 (float32): lr * sqrt(1 - beta_2^t) / (1 - beta_1^t)
__device__ __forceinline__ float adam_alpha(const AdamHp& h, long long it) {
  const float t = (float)(it + 1);
  return h.lr * (sqrtf(1.f - powf(h.b2, t)) / (1.f - powf(h.b1, t)));
}

// G[t] = the sum, in entry order, of the gradients of the entries whose table row is t; entry e owns row t when
// no earlier entry has it; t = -1 is no entry.  G is zero on entry (table_adam_kernel clears what it reads).
__global__ void table_grad_kernel(const int32_t* __restrict__ trow, const float* __restrict__ gemb, int n,
                                  int EP, float* __restrict__ G) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int t = trow[e];
  if (t < 0) return;                                  // no entry (a missing genre)
  for (int j = 0; j < e; ++j)
    if (trow[j] == t) return;
  float* g = G + (size_t)t * EP;
  for (int j = e; j < n; ++j) {
    if (trow[j] != t) continue;
    for (int k = 0; k < EP; ++k) g[k] = __fadd_rn(g[k], gemb[(size_t)j * EP + k]);
  }
}

// Keras Adam on every element of an array whose gradient table_grad_kernel deduped into G (cleared behind it):
// kApplyAdam = false, _resource_apply_sparse (the embedding tables): m = b1 m + (1-b1) G, v = b2 v + (1-b2) G^2;
// kApplyAdam = true, ApplyAdam's dense form (the one-hot rows): m += (G - m)(1-b1), v += (G^2 - v)(1-b2).
// Then w -= alpha m / (sqrt(v) + eps).  Each operation is rounded on its own (no contraction).
template <bool kApplyAdam>
__global__ void table_adam_kernel(float* __restrict__ w, float* __restrict__ m, float* __restrict__ v,
                                  float* __restrict__ G, int64_t n, AdamHp h, const long long* __restrict__ it) {
  const float alpha = adam_alpha(h, *it);
  const float c1 = 1.f - h.b1, c2 = 1.f - h.b2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float g = G[i];
    if (g != 0.f) G[i] = 0.f;
    const float mi = kApplyAdam ? __fadd_rn(m[i], __fmul_rn(__fsub_rn(g, m[i]), c1))
                                : __fadd_rn(__fmul_rn(h.b1, m[i]), __fmul_rn(c1, g));
    const float vi = kApplyAdam ? __fadd_rn(v[i], __fmul_rn(__fsub_rn(__fmul_rn(g, g), v[i]), c2))
                                : __fadd_rn(__fmul_rn(h.b2, v[i]), __fmul_rn(c2, __fmul_rn(g, g)));
    m[i] = mi;
    v[i] = vi;
    w[i] = __fsub_rn(w[i], __fdiv_rn(__fmul_rn(alpha, mi), __fadd_rn(__fsqrt_rn(vi), h.eps)));
  }
}

// the Dense gradients (CTA partials in CTA order), then TF's fused ApplyAdam: m += (g - m)(1-b1),
// v += (g^2 - v)(1-b2), w -= alpha m / (sqrt(v) + eps); then iterations += 1
__global__ void __launch_bounds__(kAdamThreads)
dense_adam_kernel(const float* __restrict__ part, int n_parts, int n, float* __restrict__ w, float* __restrict__ m,
                  float* __restrict__ v, AdamHp h, long long* it) {
  const float alpha = adam_alpha(h, *it);
  const float c1 = 1.f - h.b1, c2 = 1.f - h.b2;
  for (int q = threadIdx.x; q < n; q += kAdamThreads) {
    float g = 0.f;
    for (int c = 0; c < n_parts; ++c) g = __fadd_rn(g, part[(size_t)c * n + q]);
    const float mi = __fadd_rn(m[q], __fmul_rn(__fsub_rn(g, m[q]), c1));
    const float vi = __fadd_rn(v[q], __fmul_rn(__fsub_rn(__fmul_rn(g, g), v[q]), c2));
    m[q] = mi;
    v[q] = vi;
    w[q] = __fsub_rn(w[q], __fdiv_rn(__fmul_rn(alpha, mi), __fadd_rn(__fsqrt_rn(vi), h.eps)));
  }
  __syncthreads();
  if (threadIdx.x == 0) *it += 1;
}

}  // namespace
}  // namespace srs

using namespace srs;

struct srs_trainer {
  srs_spec spec{};
  int device = 0;
  int EP = 0, HP = 0;
  int blob_floats = 0;
  AdamHp hp{};
  Placement place;                    // where the Keras tensors live in tab, blob and fo
  NcfParams ncf{};                    // the serving parameters over the trainer's arrays (NeuralCF)
  DeepFmParams fm{};                  //   (DeepFM)
  EmbMlpParams emb{};                 //   (Wide&Deep)
  DeepFm2Params fm2{};                //   (DeepFM_v2)
  DienParams dien{};                  //   (DIEN: the step kernel's view; DIEN has no serving forward here)
  int n_ent = 0, n_fent = 0;          // table and one-hot entries per row of a step (n_fent 0: no one-hot rows)
  int genre_cols = 0;                 // the dataset's genre columns checked, 0: no genres or numerics read
  bool rated = false;                 // userRatedMovie1 read
  int (*ctas)(int B) = nullptr;       // the step's CTAs at B rows
  cudaError_t (*permute)(const TrainRows&, const TrainRows&, const int32_t*, int, cudaStream_t) = nullptr;
                                      // each epoch's rows in its order; null: the step reads through the order
  int64_t tab_floats = 0;             // (sum of the tables' rows) * EP
  float* tab[4] = {};                 // w, m, v, G   [rows][EP], padding zero
  float* blob[3] = {};                // w, m, v      [blob_floats]
  int64_t onehot = 0;                 // the one-hot rows: DeepFM's dense_2/kernel and DeepFM_v2's first_cat/kernel
                                      // (fm1_width), Wide&Deep's wide rows of dense_2/kernel
  float* fo[4] = {};                  // w, m, v, G   [onehot]
  int adam_blocks = 0, fo_blocks = 0; // the grids of table_adam_kernel over tab and over fo
  long long* d_it = nullptr;          // Adam's iteration counter, on the device
  int64_t iterations = 0;             // its host mirror
  cudaStream_t stream = nullptr;
};

namespace {

void trainer_free(srs_trainer* t) {
  if (!t) return;
  cudaSetDevice(t->device);
  for (float* p : t->tab) cudaFree(p);
  for (float* p : t->blob) cudaFree(p);
  for (float* p : t->fo) cudaFree(p);
  cudaFree(t->d_it);
  if (t->stream) cudaStreamDestroy(t->stream);
  delete t;
}

// ---- each model's facts: one block per decision -----------------------------------------------------------------

// the shapes the model's step kernel trains
int check_shape(const srs_spec& s) {
  switch (s.kind) {
    case SRS_DEEPFM:
      if (s.n_hidden != 2) return failf(SRS_ERR_INVALID, "DeepFM's fit needs exactly 2 hidden layers");
      if (s.n_genres < 1) return failf(SRS_ERR_INVALID, "empty genre vocabulary");
      for (int i = 0; i < 2; ++i)
        if (s.hidden[i] < 1 || s.hidden[i] > 64) return failf(SRS_ERR_INVALID, "DeepFM's hidden widths must be in 1..64");
      return SRS_OK;
    case SRS_WIDENDEEP:
      if (s.n_hidden != 2) return failf(SRS_ERR_INVALID, "Wide&Deep's fit needs exactly 2 hidden layers");
      if (s.n_genres < 1) return failf(SRS_ERR_INVALID, "empty genre vocabulary");
      if (s.cross_buckets < 1) return failf(SRS_ERR_INVALID, "Wide&Deep needs cross_buckets >= 1");
      for (int i = 0; i < 2; ++i)
        if (s.hidden[i] < 1 || s.hidden[i] > 128)
          return failf(SRS_ERR_INVALID, "Wide&Deep's hidden widths must be in 1..128");
      return SRS_OK;
    case SRS_DEEPFM_V2:
      if (s.n_hidden != 2) return failf(SRS_ERR_INVALID, "DeepFM_v2's fit needs exactly 2 hidden layers");
      if (s.proj_dim != 64) return failf(SRS_ERR_INVALID, "DeepFM_v2's fit needs proj_dim 64");
      if (s.n_genres < 1) return failf(SRS_ERR_INVALID, "empty genre vocabulary");
      if (s.hidden[0] < 1 || s.hidden[0] > 32 || s.hidden[1] < 1 || s.hidden[1] > 16)
        return failf(SRS_ERR_INVALID, "DeepFM_v2's hidden widths must be in 1..32 and 1..16");
      return SRS_OK;
    case SRS_DIEN:
      if (s.emb_dim > 32) return failf(SRS_ERR_INVALID, "DIEN's fit needs emb_dim in 1..32");
      if (s.hist_len < 1 || s.hist_len > kDienMaxT)
        return failf(SRS_ERR_INVALID, "DIEN's fit needs hist_len in 1..%d", kDienMaxT);
      if (s.au_hidden != 32) return failf(SRS_ERR_INVALID, "DIEN's fit needs au_hidden 32");
      if (s.n_hidden != 2) return failf(SRS_ERR_INVALID, "DIEN's fit needs exactly 2 hidden layers");
      if (s.n_genres < 1) return failf(SRS_ERR_INVALID, "empty genre vocabulary");
      if (s.hidden[0] < 1 || s.hidden[0] > 128 || s.hidden[1] < 1 || s.hidden[1] > 64)
        return failf(SRS_ERR_INVALID, "DIEN's hidden widths must be in 1..128 and 1..64");
      return SRS_OK;
    case SRS_TWOTOWERS:
      if (!s.final_dense)
        return failf(SRS_ERR_INVALID, "the two-tower model trains only with its final Dense (final_dense): without it "
                     "the output is the raw Dot, on which binary cross-entropy is not defined");
      [[fallthrough]];
    default:
      if (s.n_hidden < 1 || s.n_hidden > 3) return failf(SRS_ERR_INVALID, "1..3 hidden layers supported");
      for (int i = 0; i < s.n_hidden; ++i)
        if (s.hidden[i] < 1 || s.hidden[i] > 32) return failf(SRS_ERR_INVALID, "hidden widths must be in 1..32");
      return SRS_OK;
  }
}

// The checks of rows the trainer reads (fit, validation, evaluate; DIEN has its own), all made before any launch.
// `what` prefixes the messages: "" or "validation data: ".  weights: null, or [n] each finite and >= 0.
int check_rows(const srs_trainer* t, const srs_batch* batch, const int32_t* labels, const float* weights,
               const char* what) {
  const srs_spec& sp = t->spec;
  const int n = batch->B;
  for (int i = 0; weights && i < n; ++i)
    if (!(weights[i] >= 0.f && weights[i] <= FLT_MAX))          // false for NaN
      return failf(SRS_ERR_INVALID, "%ssample weight of row %d is %g: weights must be finite and >= 0", what, i,
                   (double)weights[i]);
  if (!batch->movie_id || !batch->user_id) return failf(SRS_ERR_INVALID, "%smovie_id and user_id are required", what);
  if (t->genre_cols && (!batch->movie_genre || !batch->user_genre || !batch->numerics ||
                        (t->rated && (!batch->hist || batch->hist_stride < 1))))
    return t->rated ? failf(SRS_ERR_INVALID, "%sWide&Deep needs movie_genre, user_genre, numerics and hist "
                            "(userRatedMovie1)", what)
                    : failf(SRS_ERR_INVALID, "%s%s needs movie_genre, user_genre and numerics", what,
                            sp.kind == SRS_DEEPFM ? "DeepFM" : "DeepFM_v2");
  for (int i = 0; i < n; ++i)
    if (labels[i] != 0 && labels[i] != 1)
      return failf(SRS_ERR_INVALID, "%slabel of row %d is %d, not 0 or 1", what, i, labels[i]);
  for (int i = 0; i < n; ++i) {
    if ((unsigned)batch->movie_id[i] >= (unsigned)sp.n_movies)
      return failf(SRS_ERR_RANGE, "%smovieId %d of row %d is outside [0, %d)", what, batch->movie_id[i], i,
                   sp.n_movies);
    if ((unsigned)batch->user_id[i] >= (unsigned)sp.n_users)
      return failf(SRS_ERR_RANGE, "%suserId %d of row %d is outside [0, %d)", what, batch->user_id[i], i,
                   sp.n_users);
  }
  for (int i = 0; t->genre_cols && i < n; ++i) {   // a negative genre is missing
    for (int k = 0; k < std::min(t->genre_cols, 3); ++k)
      if (batch->movie_genre[(size_t)i * 3 + k] >= sp.n_genres)
        return failf(SRS_ERR_RANGE, "%smovieGenre%d index %d of row %d is outside [0, %d)", what, k + 1,
                     batch->movie_genre[(size_t)i * 3 + k], i, sp.n_genres);
    for (int k = 0; k < t->genre_cols; ++k)
      if (batch->user_genre[(size_t)i * 5 + k] >= sp.n_genres)
        return failf(SRS_ERR_RANGE, "%suserGenre%d index %d of row %d is outside [0, %d)", what, k + 1,
                     batch->user_genre[(size_t)i * 5 + k], i, sp.n_genres);
    if (!t->rated) continue;
    const int m = batch->hist[(size_t)i * batch->hist_stride];
    if ((unsigned)m >= (unsigned)sp.n_movies)
      return failf(SRS_ERR_RANGE, "%suserRatedMovie1 %d of row %d is outside [0, %d)", what, m, i, sp.n_movies);
  }
  return SRS_OK;
}

// n rows of the columns the trainer's model reads on the device, and the weights when `weighted`; the others stay
// null
cudaError_t alloc_rows(Scratch& sc, const srs_trainer* t, size_t n, bool weighted, TrainRows* r) {
  *r = TrainRows{};
  cudaError_t e = sc.alloc(&r->movie, n);
  if (e == cudaSuccess && t->rated) e = sc.alloc(&r->rated, n);
  if (e == cudaSuccess) e = sc.alloc(&r->user, n);
  if (e == cudaSuccess && t->genre_cols) e = sc.alloc(&r->mgenre, n * 3);
  if (e == cudaSuccess && t->genre_cols) e = sc.alloc(&r->ugenre, n * 5);
  if (e == cudaSuccess && t->genre_cols) e = sc.alloc(&r->numerics, n * kNumNumerics);
  if (e == cudaSuccess) e = sc.alloc(&r->label, n);
  if (e == cudaSuccess && weighted) e = sc.alloc(&r->weight, n);
  return e;
}

// ---- what every model shares ----------------------------------------------------------------------------------

// rows [off, off + B) of r as a batch, with its outputs
BatchView view(const TrainRows& r, int off, int B, float* probs, float* logits, int* err) {
  BatchView b{};
  b.B = B;
  b.movie_id = r.movie + off; b.user_id = r.user + off;
  if (r.mgenre) {
    b.movie_genre = r.mgenre + (size_t)off * 3; b.user_genre = r.ugenre + (size_t)off * 5;
    b.numerics = r.numerics + (size_t)off * kNumNumerics;
  }
  if (r.rated) { b.hist = r.rated + off; b.hist_stride = 1; }
  b.probs = probs; b.logits = logits; b.err_flag = err;
  return b;
}

// batch->B rows on the device, uploaded on s: the columns the trainer's model reads, the labels and (not null) the
// weights
cudaError_t upload_rows(Scratch& sc, const srs_trainer* t, const srs_batch* b, const int32_t* labels,
                        const float* weights, TrainRows* r, cudaStream_t s) {
  const size_t n = (size_t)b->B;
  cudaError_t e = alloc_rows(sc, t, n, weights != nullptr, r);
  if (weights && e == cudaSuccess) e = cudaMemcpyAsync(r->weight, weights, n * 4, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(r->movie, b->movie_id, n * 4, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(r->user, b->user_id, n * 4, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(r->label, labels, n * 4, cudaMemcpyHostToDevice, s);
  if (r->mgenre && e == cudaSuccess)
    e = cudaMemcpyAsync(r->mgenre, b->movie_genre, n * 3 * 4, cudaMemcpyHostToDevice, s);
  if (r->ugenre && e == cudaSuccess)
    e = cudaMemcpyAsync(r->ugenre, b->user_genre, n * 5 * 4, cudaMemcpyHostToDevice, s);
  if (r->numerics && e == cudaSuccess)
    e = cudaMemcpyAsync(r->numerics, b->numerics, n * kNumNumerics * 4, cudaMemcpyHostToDevice, s);
  if (r->rated && e == cudaSuccess)
    e = cudaMemcpy2DAsync(r->rated, 4, b->hist, (size_t)b->hist_stride * 4, 4, n, cudaMemcpyHostToDevice, s);
  return e;
}

// `model.evaluate` of the trainer's current weights over n device rows, two launches on s: the serving forward, then
// one metrics_update_kernel over all the rows into em (and, with r.weight, the weighted sums into wm through wred)
cudaError_t eval_rows(const srs_trainer* t, const TrainRows& r, int n, float* probs, float* logits, int* err,
                      MetricsState* em, MetricsWeighted* wm, MetricsWeightedReduce* wred, cudaStream_t s) {
  const BatchView b = view(r, 0, n, probs, logits, err);
  cudaError_t e;
  switch (t->spec.kind) {
    case SRS_DEEPFM: e = launch_deepfm(t->fm, b, s); break;
    case SRS_WIDENDEEP: e = launch_embmlp(t->emb, b, s); break;
    case SRS_DEEPFM_V2: e = launch_deepfm2(t->fm2, b, s); break;
    default: e = launch_ncf(t->ncf, b, s); break;
  }
  if (e != cudaSuccess) return e;
  if (r.weight)
    return launch_metrics_update_weighted(probs, logits, r.label, r.weight, n, &em->cnt, &em->red, &em->loss, wm,
                                          wred, 1, s);
  return launch_metrics_update(probs, logits, r.label, n, &em->cnt, &em->red, &em->loss, 1, s);
}

// The step of the trainer's model (not DIEN) over rows [off, off + B) of an epoch: the tile models read the
// epoch's permuted rows, NeuralCF and two towers the dataset through `order` (the epoch's).  Points io.label at the
// step's labels and, weighted, io.weight at the step's weights (NeuralCF and two towers: written by the step into
// `weights`).
cudaError_t launch_step(const srs_trainer* t, const TrainRows& src, const TrainRows& rows, const int32_t* order,
                        int off, int B, int32_t* labels, float* weights, StepIO& io, cudaStream_t s) {
  if (t->spec.kind == SRS_NEURALCF || t->spec.kind == SRS_TWOTOWERS) {
    const NcfStepArgs a{t->tab[0], t->blob[0], src.movie, src.user, src.label, order + off, B, t->spec.n_movies,
                        io.b.probs, io.b.logits, labels, io.trow, io.gemb, io.part, src.weight, weights};
    io.label = labels;
    io.weight = src.weight ? weights : nullptr;
    return t->spec.kind == SRS_TWOTOWERS ? launch_twotowers_train_step(&a, t->ncf, s)
                                         : launch_ncf_train_step(&a, t->ncf, s);
  }
  io.b = view(rows, off, B, io.b.probs, io.b.logits, io.b.err_flag);
  io.label = rows.label + off;
  io.weight = rows.weight ? rows.weight + off : nullptr;
  switch (t->spec.kind) {
    case SRS_DEEPFM: {                                 // the tables come first in the placement
      DeepFmStepArgs a{t->fm, io, {}};
      for (int k = 0; k < kDeepFmTables; ++k) a.tab_row0[k] = t->place[k].table_row;
      return launch_deepfm_train_step(t->EP, &a, s);
    }
    case SRS_WIDENDEEP: {
      WideDeepStepArgs a{t->emb, io, {}};
      for (int k = 0; k < kWideDeepTables; ++k) a.tab_row0[k] = t->place[kEmbMlpSlotTable[k]].table_row;
      return launch_widendeep_train_step(t->EP, &a, s);
    }
    default: {
      DeepFm2StepArgs a{t->fm2, io, {}};
      for (int k = 0; k < kDeepFm2Tables; ++k) a.tab_row0[k] = t->place[k].table_row;
      return launch_deepfm2_train_step(t->EP, &a, s);
    }
  }
}

// The update after a step of B rows, in this order: table_grad_kernel over its table entries and (models with
// one-hot rows) at width 1 over its one-hot entries, table_adam_kernel<false> over the tables and <true> over the
// one-hot rows, dense_adam_kernel over the step's CTA partials
cudaError_t update(srs_trainer* t, const StepIO& io, int B, cudaStream_t s) {
  const int n_ent = t->n_ent * B, n_fent = t->n_fent * B;
  table_grad_kernel<<<(n_ent + 127) / 128, 128, 0, s>>>(io.trow, io.gemb, n_ent, t->EP, t->tab[3]);
  if (n_fent) table_grad_kernel<<<(n_fent + 127) / 128, 128, 0, s>>>(io.frow, io.fgrad, n_fent, 1, t->fo[3]);
  table_adam_kernel<false><<<t->adam_blocks, 256, 0, s>>>(t->tab[0], t->tab[1], t->tab[2], t->tab[3], t->tab_floats,
                                                          t->hp, t->d_it);
  if (n_fent)
    table_adam_kernel<true><<<t->fo_blocks, 256, 0, s>>>(t->fo[0], t->fo[1], t->fo[2], t->fo[3], t->onehot, t->hp,
                                                         t->d_it);
  dense_adam_kernel<<<1, kAdamThreads, 0, s>>>(io.part, t->ctas(B), t->blob_floats, t->blob[0], t->blob[1],
                                               t->blob[2], t->hp, t->d_it);
  g_launch_count += n_fent ? 5 : 3;
  return cudaGetLastError();
}

int check_fit_sizes(int n, int batch_size, int epochs) {
  if (n < 1) return failf(SRS_ERR_INVALID, "fit needs at least one row");
  if (batch_size < 1) return failf(SRS_ERR_INVALID, "batch_size must be at least 1");
  if (epochs < 1) return failf(SRS_ERR_INVALID, "epochs must be at least 1");
  return SRS_OK;
}

// each epoch's [n] of the [epochs][n] order is a permutation of 0..n-1
int check_orders(const int32_t* order, int n, int epochs) {
  std::vector<char> seen(n);
  for (int e = 0; e < epochs; ++e) {
    std::fill(seen.begin(), seen.end(), 0);
    for (int i = 0; i < n; ++i) {
      const int r = order[(size_t)e * n + i];
      if (r < 0 || r >= n || seen[r]) return failf(SRS_ERR_INVALID, "order of epoch %d is not a permutation of 0..%d", e, n - 1);
      seen[r] = 1;
    }
  }
  return SRS_OK;
}

// A fit's device buffers that every model has: the order uploaded, each epoch's metrics state zeroed, and a
// step's outputs and entry lists for up to Bmax rows; a weighted fit's weighted metrics and the step's weights
struct FitBuffers {
  int32_t* order;                     // [epochs][n]
  MetricsState* met;                  // [epochs]
  int32_t* labels;                    // [Bmax] the step's labels (NeuralCF, DIEN: written by the step)
  StepIO io;                          // b.probs, b.logits, trow, gemb, part and (one-hot rows) frow, fgrad
  MetricsWeighted* wmet;              // [epochs] weighted only, zeroed
  MetricsWeightedReduce* wred;        //   its CTA partials (shared with validation: one stream)
  float* weights;                     //   [Bmax] the step's weights (NeuralCF, two towers: written by the step)
};

cudaError_t alloc_fit(Scratch& sc, const srs_trainer* t, const int32_t* order, int n, int epochs, int Bmax,
                      bool weighted, FitBuffers* f, cudaStream_t s) {
  *f = FitBuffers{};
  const size_t ent = (size_t)t->n_ent * Bmax, fent = (size_t)t->n_fent * Bmax;
  cudaError_t e = sc.alloc(&f->order, (size_t)epochs * n);
  if (e == cudaSuccess) e = sc.alloc(&f->met, epochs);
  if (e == cudaSuccess) e = sc.alloc(&f->labels, Bmax);
  if (e == cudaSuccess) e = sc.alloc(&f->io.b.probs, Bmax);
  if (e == cudaSuccess) e = sc.alloc(&f->io.b.logits, Bmax);
  if (e == cudaSuccess) e = sc.alloc(&f->io.trow, ent);
  if (e == cudaSuccess) e = sc.alloc(&f->io.gemb, ent * t->EP);
  if (e == cudaSuccess) e = sc.alloc(&f->io.part, (size_t)t->ctas(Bmax) * t->blob_floats);
  if (e == cudaSuccess && fent) e = sc.alloc(&f->io.frow, fent);
  if (e == cudaSuccess && fent) e = sc.alloc(&f->io.fgrad, fent);
  if (e == cudaSuccess) e = cudaMemcpyAsync(f->order, order, (size_t)epochs * n * 4, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemsetAsync(f->met, 0, sizeof(MetricsState) * epochs, s);
  if (e == cudaSuccess && weighted) e = sc.alloc(&f->wmet, epochs);
  if (e == cudaSuccess && weighted) e = sc.alloc(&f->wred, 1);
  if (e == cudaSuccess && weighted) e = sc.alloc(&f->weights, Bmax);
  if (e == cudaSuccess && weighted) e = cudaMemsetAsync(f->wmet, 0, sizeof(MetricsWeighted) * epochs, s);
  return e;
}

// A DIEN trainer at an entry point of the other models: its fit takes negatives and reports DIEN's own metrics
int dien_rejected(const char* what) {
  return failf(SRS_ERR_INVALID, "a DIEN trainer's %s is srs_trainer_fit_dien_host: DIEN trains on negatives and "
               "reports its own loss, auc and auc_value (a trained model's evaluate is srs_dien_evaluate_host_batches)",
               what);
}

// The trainer of any trainable kind (the entry points below check the kind against their own lists first)
int trainer_create(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                   const srs_adam* hp, srs_trainer** out) {
  const srs_spec& s = *spec;
  if (s.emb_dim < 1 || s.emb_dim > 64) return failf(SRS_ERR_INVALID, "emb_dim must be in 1..64");
  if (s.n_movies < 1 || s.n_users < 1) return failf(SRS_ERR_INVALID, "empty vocabulary");
  PROPAGATE(check_shape(s));
  AdamHp h{0.001f, 0.9f, 0.999f, 1e-7f};              // Keras's Adam defaults
  if (hp) h = AdamHp{hp->lr, hp->beta_1, hp->beta_2, hp->epsilon};
  if (!(h.lr > 0.f && h.lr < 1e30f) || !(h.b1 >= 0.f && h.b1 < 1.f) || !(h.b2 >= 0.f && h.b2 < 1.f) ||
      !(h.eps > 0.f && h.eps < 1e30f))
    return failf(SRS_ERR_INVALID, "Adam needs lr > 0, 0 <= beta_1, beta_2 < 1 and epsilon > 0");
  if (n_tensors < 0 || (n_tensors > 0 && !tensors)) return failf(SRS_ERR_INVALID, "null tensors");
  PROPAGATE(check_device(device));

  srs_trainer* t = new srs_trainer();
  t->spec = s;
  t->device = device;
  t->hp = h;
  t->EP = round_ep(s.emb_dim);
  const int EP = t->EP;
  switch (s.kind) {         // placement, HP, the blob, the one-hot rows, the entries per row and the dataset's columns
    case SRS_DEEPFM:
      t->HP = 64;
      t->place = place_deepfm(s, EP, &t->fm);
      t->blob_floats = DeepFmBlob::of(EP).floats;
      t->onehot = (int64_t)2 * s.n_genres + s.n_movies + s.n_users;
      t->n_ent = kDeepFmTables, t->n_fent = 4, t->genre_cols = 1;
      t->ctas = deepfm_train_ctas, t->permute = launch_deepfm_permute;
      break;
    case SRS_WIDENDEEP:
      t->HP = 128;
      t->place = place_embmlp(s, EP, &t->emb);
      t->blob_floats = EmbMlpBlob::of(EP).floats;
      t->onehot = s.cross_buckets;
      t->n_ent = kWideDeepTables, t->n_fent = 1, t->genre_cols = 5, t->rated = true;
      t->ctas = widendeep_train_ctas, t->permute = launch_widendeep_permute;
      break;
    case SRS_DEEPFM_V2:                                  // DeepFM's columns, permuted as DeepFM's
      t->place = place_deepfm2(s, EP, &t->fm2);
      t->blob_floats = DeepFm2Blob::of(EP).floats;
      t->onehot = (int64_t)2 * s.n_genres + s.n_movies + s.n_users;
      t->n_ent = kDeepFm2Tables, t->n_fent = 4, t->genre_cols = 1;
      t->ctas = deepfm2_train_ctas, t->permute = launch_deepfm_permute;
      break;
    case SRS_DIEN:                                       // its fit checks and uploads its own columns
      t->place = place_dien(s, EP, true, &t->dien);   // the auxiliary head is part of the objective
      t->blob_floats = DienLayout::of(EP).floats;
      t->n_ent = 2 * s.hist_len + 3;
      t->ctas = dien_train_ctas;
      break;
    default:                                             // NeuralCF and two towers
      t->HP = *std::max_element(s.hidden, s.hidden + s.n_hidden) <= 16 ? 16 : 32;
      t->place = place_ncf(s, EP, t->HP, &t->ncf);
      t->blob_floats = t->ncf.blob_floats;
      t->n_ent = 2;
      t->ctas = s.kind == SRS_TWOTOWERS ? twotowers_train_ctas : ncf_train_ctas;
      break;
  }
  t->tab_floats = table_rows(t->place) * EP;
  const int nb = t->blob_floats;

  // every tensor looked up, and the Dense ones placed, before the first device call
  std::vector<float> blob(nb, 0.f), onehot(t->onehot, 0.f);
  std::vector<const float*> src;                       // each tensor's data, in placement order
  TensorLookup lookup(tensors, n_tensors);
  for (const Placed& x : t->place) {
    src.push_back(lookup.host(x.name.c_str(), x.rows, x.cols));
    if (!src.back()) { delete t; return lookup.status; }
    scatter(x, src.back(), blob.data(), onehot.data());
  }

  // the shared memory opt-ins are per device: the serving forwards' that validation and evaluate run (deepfm_kernel,
  // deepfm2_kernel, embmlp_kernel), as srs_model_create makes them, and the step's, at its largest size, so that a
  // later trainer on the device never lowers it
  cudaError_t ce = cudaSetDevice(device);
  if (ce == cudaSuccess) ce = setup_deepfm_attributes();
  if (ce == cudaSuccess) ce = setup_embmlp_attributes();
  if (ce == cudaSuccess) {
    switch (s.kind) {
      case SRS_DEEPFM: ce = launch_deepfm_train_step(EP, nullptr, nullptr); break;
      case SRS_WIDENDEEP: ce = launch_widendeep_train_step(EP, nullptr, nullptr); break;
      case SRS_DEEPFM_V2: ce = launch_deepfm2_train_step(EP, nullptr, nullptr); break;
      case SRS_DIEN: ce = launch_dien_train_step(EP, nullptr, nullptr); break;
      case SRS_TWOTOWERS: ce = launch_twotowers_train_step(nullptr, t->ncf, nullptr); break;
      default: ce = launch_ncf_train_step(nullptr, t->ncf, nullptr); break;
    }
  }
  if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&t->stream, cudaStreamNonBlocking);
  for (int k = 0; k < 4 && ce == cudaSuccess; ++k) ce = cudaMalloc(&t->tab[k], t->tab_floats * sizeof(float));
  for (int k = 0; k < 3 && ce == cudaSuccess; ++k) ce = cudaMalloc(&t->blob[k], (size_t)nb * sizeof(float));
  for (int k = 0; k < 4 && ce == cudaSuccess && t->onehot; ++k) ce = cudaMalloc(&t->fo[k], t->onehot * sizeof(float));
  if (ce == cudaSuccess) ce = cudaMalloc(&t->d_it, sizeof(long long));
  for (int k = 0; k < 4 && ce == cudaSuccess; ++k) ce = cudaMemset(t->tab[k], 0, t->tab_floats * sizeof(float));
  for (int k = 1; k < 3 && ce == cudaSuccess; ++k) ce = cudaMemset(t->blob[k], 0, (size_t)nb * sizeof(float));
  for (int k = 1; k < 4 && ce == cudaSuccess && t->onehot; ++k) ce = cudaMemset(t->fo[k], 0, t->onehot * sizeof(float));
  if (ce == cudaSuccess) ce = cudaMemset(t->d_it, 0, sizeof(long long));
  if (ce == cudaSuccess) ce = cudaMemcpy(t->blob[0], blob.data(), (size_t)nb * sizeof(float), cudaMemcpyHostToDevice);
  if (ce == cudaSuccess && t->onehot)
    ce = cudaMemcpy(t->fo[0], onehot.data(), t->onehot * sizeof(float), cudaMemcpyHostToDevice);
  for (size_t k = 0; k < t->place.size() && ce == cudaSuccess; ++k) {   // [V][E] -> [V][EP], padding stays zero
    const Placed& x = t->place[k];
    if (x.table_row < 0) continue;
    ce = cudaMemcpy2D(t->tab[0] + x.table_row * EP, (size_t)EP * sizeof(float), src[k], (size_t)x.cols * sizeof(float),
                      (size_t)x.cols * sizeof(float), (size_t)x.rows, cudaMemcpyHostToDevice);
  }
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  if (ce != cudaSuccess) {
    trainer_free(t);
    return failf(ce == cudaErrorMemoryAllocation ? SRS_ERR_NOMEM : SRS_ERR_CUDA, "trainer setup failed: %s",
                 cudaGetErrorString(ce));
  }
  // the serving parameters over the trainer's arrays; every placement puts its tables first
  static_assert(kWideDeepTables >= kDeepFmTables && kWideDeepTables >= kDeepFm2Tables &&
                kWideDeepTables >= kDienTables, "tables[] holds every model's tables");
  const float* tables[kWideDeepTables] = {};
  for (int k = 0; k < kWideDeepTables && k < (int)t->place.size() && t->place[k].table_row >= 0; ++k)
    tables[k] = t->tab[0] + t->place[k].table_row * EP;
  switch (s.kind) {
    case SRS_DEEPFM:
      t->fm.fm_movie = tables[0]; t->fm.fm_user = tables[1]; t->fm.fm_mgenre = tables[2]; t->fm.fm_ugenre = tables[3];
      t->fm.deep_movie = tables[4]; t->fm.deep_user = tables[5];
      point_into_blob(&t->fm, t->blob[0]);
      t->fm.first = t->fo[0];
      break;
    case SRS_WIDENDEEP:
      point_into_blob(&t->emb, tables, t->blob[0]);
      t->emb.wide = t->fo[0];
      break;
    case SRS_DEEPFM_V2:
      point_into_blob(&t->fm2, tables, t->blob[0]);
      t->fm2.first = t->fo[0];
      break;
    case SRS_DIEN:
      point_into_blob(&t->dien, tables, t->blob[0], blob.data());   // the step kernel reads b3 from the blob
      break;
    default:
      t->ncf.movie = tables[0]; t->ncf.user = tables[1]; t->ncf.blob = t->blob[0];
      break;
  }
  int dev_sms = 132;
  cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, device);
  t->adam_blocks = (int)std::min<int64_t>((t->tab_floats + 255) / 256, (int64_t)dev_sms * 8);
  t->fo_blocks = (int)std::min<int64_t>((t->onehot + 255) / 256, (int64_t)dev_sms * 8);
  *out = t;
  return SRS_OK;
}

}  // namespace

extern "C" {

// NeuralCF and DeepFM only, as this entry point has always been documented
int srs_trainer_create(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                       const srs_adam* hp, srs_trainer** out) {
  if (!spec || !out) return failf(SRS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (spec->kind != SRS_NEURALCF && spec->kind != SRS_DEEPFM)
    return failf(SRS_ERR_INVALID, "srs_trainer_create trains NeuralCF (neural_cf_model_1) and DeepFM only; "
                 "srs_trainer_create_ex also trains Wide&Deep");
  return trainer_create(spec, tensors, n_tensors, device, hp, out);
}

// NeuralCF, DeepFM and Wide&Deep, as this entry point has always been documented
int srs_trainer_create_ex(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                          const srs_adam* hp, srs_trainer** out) {
  if (!spec || !out) return failf(SRS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (spec->kind != SRS_NEURALCF && spec->kind != SRS_DEEPFM && spec->kind != SRS_WIDENDEEP)
    return failf(SRS_ERR_INVALID, "fit is implemented for NeuralCF (neural_cf_model_1), DeepFM and Wide&Deep only; "
                 "srs_trainer_create_any trains every kind this library can train");
  return trainer_create(spec, tensors, n_tensors, device, hp, out);
}

// every kind this library can train; the list grows with the library
int srs_trainer_create_any(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                           const srs_adam* hp, srs_trainer** out) {
  if (!spec || !out) return failf(SRS_ERR_INVALID, "null argument");
  *out = nullptr;
  const int k = spec->kind;
  if (k != SRS_NEURALCF && k != SRS_TWOTOWERS && k != SRS_DEEPFM && k != SRS_WIDENDEEP && k != SRS_DEEPFM_V2 &&
      k != SRS_DIEN)
    return failf(SRS_ERR_INVALID, "fit is implemented for NeuralCF (neural_cf_model_1), two towers "
                 "(neural_cf_model_2), DeepFM, Wide&Deep, DeepFM_v2 and DIEN only");
  return trainer_create(spec, tensors, n_tensors, device, hp, out);
}

void srs_trainer_destroy(srs_trainer* t) { trainer_free(t); }

int64_t srs_trainer_iterations(const srs_trainer* t) { return t ? t->iterations : 0; }

int srs_trainer_fit_host(srs_trainer* t, const srs_batch* batch, const int32_t* labels, const int32_t* order,
                         int32_t batch_size, int32_t epochs, srs_eval_result* history) {
  return srs_trainer_fit_validate_host(t, batch, labels, order, batch_size, epochs, history, nullptr, nullptr, 1,
                                       nullptr);
}

int srs_trainer_fit_validate_host(srs_trainer* t, const srs_batch* batch, const int32_t* labels, const int32_t* order,
                                  int32_t batch_size, int32_t epochs, srs_eval_result* history,
                                  const srs_batch* val_batch, const int32_t* val_labels, int32_t val_freq,
                                  srs_eval_result* val_history) {
  return srs_trainer_fit_weighted_host(t, batch, labels, nullptr, order, batch_size, epochs, history, val_batch,
                                       val_labels, nullptr, val_freq, val_history);
}

int srs_trainer_fit_weighted_host(srs_trainer* t, const srs_batch* batch, const int32_t* labels, const float* weights,
                                  const int32_t* order, int32_t batch_size, int32_t epochs, srs_eval_result* history,
                                  const srs_batch* val_batch, const int32_t* val_labels, const float* val_weights,
                                  int32_t val_freq, srs_eval_result* val_history) {
  if (!t || !batch || !labels || !order) return failf(SRS_ERR_INVALID, "null argument");
  if (t->spec.kind == SRS_DIEN) return dien_rejected("fit");
  const int n = batch->B;
  // every check before the first launch: a rejected call leaves the trainer as it was
  PROPAGATE(check_fit_sizes(n, batch_size, epochs));
  PROPAGATE(check_rows(t, batch, labels, weights, ""));
  PROPAGATE(check_orders(order, n, epochs));
  const int nv = val_batch ? val_batch->B : 0;         // validation rows; 0: no validation
  if (val_batch) {
    if (!val_labels) return failf(SRS_ERR_INVALID, "validation data: null labels");
    if (nv < 1) return failf(SRS_ERR_INVALID, "validation data: needs at least one row");
    if (val_freq < 1) return failf(SRS_ERR_INVALID, "validation_freq must be at least 1");
    PROPAGATE(check_rows(t, val_batch, val_labels, val_weights, "validation data: "));
  }
  const bool vweighted = nv && val_weights;
  CUDA_TRY(cudaSetDevice(t->device));
  cudaStream_t s = t->stream;
  Scratch sc;
  FitBuffers f;
  CUDA_TRY(alloc_fit(sc, t, order, n, epochs, std::min(batch_size, n), weights != nullptr, &f, s));
  TrainRows src{}, rows{};                             // the dataset, and (the tile models) the epoch's rows in order
  CUDA_TRY(upload_rows(sc, t, batch, labels, weights, &src, s));
  if (t->permute) CUDA_TRY(alloc_rows(sc, t, n, weights != nullptr, &rows));
  CUDA_TRY(sc.alloc(&f.io.b.err_flag, 1));
  CUDA_TRY(cudaMemsetAsync(f.io.b.err_flag, 0, sizeof(int), s));
  // validation: its rows uploaded once, in file order; each validated epoch's metrics in its own state
  TrainRows vrows{};
  float *d_vprobs = nullptr, *d_vlogits = nullptr;
  MetricsState* d_vmet = nullptr;
  MetricsWeighted* d_vwmet = nullptr;
  if (nv) {
    CUDA_TRY(upload_rows(sc, t, val_batch, val_labels, vweighted ? val_weights : nullptr, &vrows, s));
    CUDA_TRY(sc.alloc(&d_vprobs, nv));
    CUDA_TRY(sc.alloc(&d_vlogits, nv));
    CUDA_TRY(sc.alloc(&d_vmet, epochs));
    CUDA_TRY(cudaMemsetAsync(d_vmet, 0, sizeof(MetricsState) * epochs, s));
  }
  if (vweighted) {
    CUDA_TRY(sc.alloc(&d_vwmet, epochs));
    CUDA_TRY(cudaMemsetAsync(d_vwmet, 0, sizeof(MetricsWeighted) * epochs, s));
    if (!f.wred) CUDA_TRY(sc.alloc(&f.wred, 1));
  }

  int64_t steps = 0;
  for (int e = 0; e < epochs; ++e) {
    const int32_t* order_e = f.order + (size_t)e * n;
    if (t->permute) CUDA_TRY(t->permute(src, rows, order_e, n, s));
    for (int off = 0; off < n; off += batch_size) {
      const int B = std::min(batch_size, n - off);
      CUDA_TRY(launch_step(t, src, rows, order_e, off, B, f.labels, f.weights, f.io, s));
      CUDA_TRY(update(t, f.io, B, s));
      if (f.io.weight)
        CUDA_TRY(launch_metrics_update_weighted(f.io.b.probs, f.io.b.logits, f.io.label, f.io.weight, B,
                                                &f.met[e].cnt, &f.met[e].red, &f.met[e].loss, &f.wmet[e], f.wred, 1,
                                                s));
      else
        CUDA_TRY(launch_metrics_update(f.io.b.probs, f.io.b.logits, f.io.label, B, &f.met[e].cnt, &f.met[e].red,
                                        &f.met[e].loss, 1, s));
      ++steps;
    }
    // after the epoch's last update, on the same stream: no host synchronisation
    if (nv && (e + 1) % val_freq == 0)
      CUDA_TRY(eval_rows(t, vrows, nv, d_vprobs, d_vlogits, f.io.b.err_flag, &d_vmet[e],
                         d_vwmet ? &d_vwmet[e] : nullptr, f.wred, s));
  }
  std::vector<MetricsState> met(epochs), vmet(nv ? epochs : 0);
  std::vector<MetricsWeighted> wmet(weights ? epochs : 0), vwmet(vweighted ? epochs : 0);
  CUDA_TRY(cudaMemcpyAsync(met.data(), f.met, sizeof(MetricsState) * epochs, cudaMemcpyDeviceToHost, s));
  if (nv) CUDA_TRY(cudaMemcpyAsync(vmet.data(), d_vmet, sizeof(MetricsState) * epochs, cudaMemcpyDeviceToHost, s));
  if (weights)
    CUDA_TRY(cudaMemcpyAsync(wmet.data(), f.wmet, sizeof(MetricsWeighted) * epochs, cudaMemcpyDeviceToHost, s));
  if (vweighted)
    CUDA_TRY(cudaMemcpyAsync(vwmet.data(), d_vwmet, sizeof(MetricsWeighted) * epochs, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  t->iterations += steps;
  for (int e = 0; e < epochs; ++e) {
    const bool validated = nv && (e + 1) % val_freq == 0;
    if (met[e].cnt.err) return failf(SRS_ERR_INVALID, "epoch %d produced a probability that is NaN or outside [0, 1]", e);
    if (validated && vmet[e].cnt.err)
      return failf(SRS_ERR_INVALID, "the validation of epoch %d produced a probability that is NaN or outside [0, 1]",
                   e);
    if (history && weights)
      metrics_summarise_weighted(met[e].cnt.hist, met[e].cnt.correct, wmet[e], met[e].loss, &history[e]);
    else if (history)
      metrics_summarise(met[e].cnt.hist, met[e].cnt.correct, met[e].loss, &history[e], nullptr);
    if (val_history) {
      val_history[e] = srs_eval_result{};
      if (validated && vweighted)
        metrics_summarise_weighted(vmet[e].cnt.hist, vmet[e].cnt.correct, vwmet[e], vmet[e].loss, &val_history[e]);
      else if (validated)
        metrics_summarise(vmet[e].cnt.hist, vmet[e].cnt.correct, vmet[e].loss, &val_history[e], nullptr);
    }
  }
  return SRS_OK;
}

int srs_trainer_evaluate_host(srs_trainer* t, const srs_batch* batch, const int32_t* labels, srs_eval_result* out) {
  return srs_trainer_evaluate_weighted_host(t, batch, labels, nullptr, out);
}

int srs_trainer_evaluate_weighted_host(srs_trainer* t, const srs_batch* batch, const int32_t* labels,
                                       const float* weights, srs_eval_result* out) {
  if (!t || !batch || !labels || !out) return failf(SRS_ERR_INVALID, "null argument");
  if (t->spec.kind == SRS_DIEN) return dien_rejected("evaluate");
  const int n = batch->B;
  if (n < 1) return failf(SRS_ERR_INVALID, "evaluate needs at least one row");
  PROPAGATE(check_rows(t, batch, labels, weights, ""));
  CUDA_TRY(cudaSetDevice(t->device));
  cudaStream_t s = t->stream;
  Scratch sc;
  TrainRows rows{};
  float *d_probs, *d_logits;
  int* d_err;
  MetricsState* d_met;
  MetricsWeighted* d_wmet = nullptr;
  MetricsWeightedReduce* d_wred = nullptr;
  CUDA_TRY(upload_rows(sc, t, batch, labels, weights, &rows, s));
  CUDA_TRY(sc.alloc(&d_probs, n));
  CUDA_TRY(sc.alloc(&d_logits, n));
  CUDA_TRY(sc.alloc(&d_err, 1));
  CUDA_TRY(sc.alloc(&d_met, 1));
  CUDA_TRY(cudaMemsetAsync(d_err, 0, sizeof(int), s));
  CUDA_TRY(cudaMemsetAsync(d_met, 0, sizeof(MetricsState), s));
  if (weights) {
    CUDA_TRY(sc.alloc(&d_wmet, 1));
    CUDA_TRY(sc.alloc(&d_wred, 1));
    CUDA_TRY(cudaMemsetAsync(d_wmet, 0, sizeof(MetricsWeighted), s));
  }
  CUDA_TRY(eval_rows(t, rows, n, d_probs, d_logits, d_err, d_met, d_wmet, d_wred, s));
  MetricsState met;
  MetricsWeighted wmet;
  CUDA_TRY(cudaMemcpyAsync(&met, d_met, sizeof(met), cudaMemcpyDeviceToHost, s));
  if (weights) CUDA_TRY(cudaMemcpyAsync(&wmet, d_wmet, sizeof(wmet), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  if (met.cnt.err) return failf(SRS_ERR_INVALID, "evaluate produced a probability that is NaN or outside [0, 1]");
  if (weights)
    metrics_summarise_weighted(met.cnt.hist, met.cnt.correct, wmet, met.loss, out);
  else
    metrics_summarise(met.cnt.hist, met.cnt.correct, met.loss, out, nullptr);
  return SRS_OK;
}

int srs_trainer_fit_dien_host(srs_trainer* t, const srs_batch* batch, const int32_t* neg_hist, int32_t neg_stride,
                              const int32_t* labels, const int32_t* order, int32_t batch_size, int32_t epochs,
                              srs_dien_eval_result* history) {
  if (!t || !batch || !labels || !order) return failf(SRS_ERR_INVALID, "null argument");
  if (t->spec.kind != SRS_DIEN)
    return failf(SRS_ERR_INVALID, "srs_trainer_fit_dien_host trains DIEN; this trainer's fit is srs_trainer_fit_host");
  const srs_spec& sp = t->spec;
  const int n = batch->B, T = sp.hist_len;
  // every check before the first launch: a rejected call leaves the trainer as it was
  PROPAGATE(check_fit_sizes(n, batch_size, epochs));
  if (!batch->movie_id || !batch->user_id || !batch->movie_genre || !batch->user_genre || !batch->numerics ||
      !batch->hist || batch->hist_stride < T)
    return failf(SRS_ERR_INVALID, "DIEN needs movie_id, user_id, movie_genre, user_genre, numerics and hist "
                 "[B][hist_stride >= %d]", T);
  if (T > 1 && (!neg_hist || neg_stride < T - 1))
    return failf(SRS_ERR_INVALID, "neg_hist [B][neg_stride >= %d] is required", T - 1);
  // a numeric column's float32, as the kernels read it; |float(raw)| <= 2^31, which int64 holds (int may not)
  auto as_id = [](int32_t raw) { return (int64_t)(float)raw; };
  for (int i = 0; i < n; ++i) {
    if (labels[i] != 0 && labels[i] != 1)
      return failf(SRS_ERR_INVALID, "label of row %d is %d, not 0 or 1", i, labels[i]);
    const int64_t m = as_id(batch->movie_id[i]);
    if (m < 0 || m >= sp.n_movies)
      return failf(SRS_ERR_RANGE, "movieId %d of row %d is outside [0, %d)", batch->movie_id[i], i, sp.n_movies);
    if ((unsigned)batch->user_id[i] >= (unsigned)sp.n_users)
      return failf(SRS_ERR_RANGE, "userId %d of row %d is outside [0, %d)", batch->user_id[i], i, sp.n_users);
    if (batch->movie_genre[(size_t)i * 3] >= sp.n_genres)   // a negative genre is missing
      return failf(SRS_ERR_RANGE, "movieGenre1 index %d of row %d is outside [0, %d)", batch->movie_genre[(size_t)i * 3],
                   i, sp.n_genres);
    if (batch->user_genre[(size_t)i * 5] >= sp.n_genres)
      return failf(SRS_ERR_RANGE, "userGenre1 index %d of row %d is outside [0, %d)", batch->user_genre[(size_t)i * 5],
                   i, sp.n_genres);
    for (int k = 0; k < T; ++k) {
      const int64_t h = as_id(batch->hist[(size_t)i * batch->hist_stride + k]);
      if (h < 0 || h >= sp.n_movies)
        return failf(SRS_ERR_RANGE, "history id %d (position %d) of row %d is outside [0, %d)",
                     batch->hist[(size_t)i * batch->hist_stride + k], k, i, sp.n_movies);
    }
    for (int k = 0; k + 1 < T; ++k) {
      const int64_t g = as_id(neg_hist[(size_t)i * neg_stride + k]);
      if (g < 0 || g >= sp.n_movies)
        return failf(SRS_ERR_RANGE, "negative movie id %d (position %d) of row %d is outside [0, %d)",
                     neg_hist[(size_t)i * neg_stride + k], k + 2, i, sp.n_movies);
    }
  }
  PROPAGATE(check_orders(order, n, epochs));
  CUDA_TRY(cudaSetDevice(t->device));
  const int Bmax = std::min(batch_size, n), K = (n + batch_size - 1) / batch_size;
  cudaStream_t s = t->stream;
  Scratch sc;
  FitBuffers f;
  CUDA_TRY(alloc_fit(sc, t, order, n, epochs, Bmax, false, &f, s));
  TrainRows src;                                       // movieId, userId and the labels
  CUDA_TRY(upload_rows(sc, t, batch, labels, nullptr, &src, s));
  int32_t *d_ug, *d_mg, *d_hist, *d_neg = nullptr;
  float *d_num, *d_aux, *d_final, *d_rec;
  double *d_bloss, *d_auc, *d_aucsum;
  unsigned long long* d_bhist;
  const size_t N = (size_t)n;
  CUDA_TRY(sc.alloc(&d_ug, N));
  CUDA_TRY(sc.alloc(&d_mg, N));
  CUDA_TRY(sc.alloc(&d_num, N * kNumNumerics));
  CUDA_TRY(sc.alloc(&d_hist, N * T));
  if (T > 1) CUDA_TRY(sc.alloc(&d_neg, N * (T - 1)));
  CUDA_TRY(sc.alloc(&d_aux, Bmax));
  CUDA_TRY(sc.alloc(&d_final, Bmax));
  CUDA_TRY(sc.alloc(&d_rec, dien_train_rec_floats(Bmax, T)));
  CUDA_TRY(sc.alloc(&d_bloss, (size_t)epochs * K));
  CUDA_TRY(sc.alloc(&d_auc, (size_t)K));
  CUDA_TRY(sc.alloc(&d_aucsum, (size_t)epochs));
  CUDA_TRY(sc.alloc(&d_bhist, (size_t)K * 2 * kMetBins));
  CUDA_TRY(cudaMemcpy2DAsync(d_ug, 4, batch->user_genre, 5 * 4, 4, N, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpy2DAsync(d_mg, 4, batch->movie_genre, 3 * 4, 4, N, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_num, batch->numerics, N * kNumNumerics * 4, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpy2DAsync(d_hist, (size_t)T * 4, batch->hist, (size_t)batch->hist_stride * 4, (size_t)T * 4, N,
                             cudaMemcpyHostToDevice, s));
  if (T > 1)
    CUDA_TRY(cudaMemcpy2DAsync(d_neg, (size_t)(T - 1) * 4, neg_hist, (size_t)neg_stride * 4, (size_t)(T - 1) * 4, N,
                               cudaMemcpyHostToDevice, s));

  DienStepArgs a{};
  a.p = t->dien;
  a.blob = t->blob[0];
  a.movie = src.movie; a.user = src.user; a.ugenre = d_ug; a.mgenre = d_mg; a.numerics = d_num;
  a.hist = d_hist; a.neg = d_neg; a.label = src.label;
  for (int k = 0; k < kDienTables; ++k) a.tab_row0[k] = t->place[k].table_row;   // the tables come first
  a.probs = f.io.b.probs; a.logits = f.io.b.logits; a.aux = d_aux; a.labels = f.labels;
  a.trow = f.io.trow; a.gemb = f.io.gemb; a.rec = d_rec; a.part = f.io.part;
  for (int e = 0; e < epochs; ++e) {
    CUDA_TRY(cudaMemsetAsync(d_bhist, 0, (size_t)K * 2 * kMetBins * sizeof(unsigned long long), s));
    for (int k = 0; k < K; ++k) {
      const int off = k * batch_size, B = std::min(batch_size, n - off);
      a.B = B;
      a.order = f.order + (size_t)e * n + off;
      CUDA_TRY(launch_dien_train_step(t->EP, &a, s));
      CUDA_TRY(update(t, f.io, B, s));
      CUDA_TRY(launch_dien_final_loss(a.logits, a.labels, d_aux, B, d_final, d_bloss + (size_t)e * K + k, s));
      CUDA_TRY(launch_metrics_update(a.probs, a.logits, a.labels, B, &f.met[e].cnt, &f.met[e].red, nullptr, 0, s,
                                      d_bhist + (size_t)k * 2 * kMetBins));
    }
    CUDA_TRY(launch_auc_value(d_bhist, K, d_auc, d_aucsum + e, s));
  }
  std::vector<MetricsState> met(epochs);
  std::vector<double> bloss((size_t)epochs * K), aucsum(epochs);
  CUDA_TRY(cudaMemcpyAsync(met.data(), f.met, sizeof(MetricsState) * epochs, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(bloss.data(), d_bloss, bloss.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaMemcpyAsync(aucsum.data(), d_aucsum, aucsum.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  t->iterations += (int64_t)epochs * K;
  for (int e = 0; e < epochs; ++e) {
    if (met[e].cnt.err) return failf(SRS_ERR_INVALID, "epoch %d produced a probability that is NaN or outside [0, 1]", e);
    if (!history) continue;
    double loss = 0.0;                                   // the batches' final_loss sums, in batch order
    for (int k = 0; k < K; ++k) loss += bloss[(size_t)e * K + k];
    srs_eval_result r{};
    metrics_summarise(met[e].cnt.hist, met[e].cnt.correct, loss, &r, nullptr);
    history[e].rows = n;
    history[e].batches = K;
    history[e].loss = r.loss;
    history[e].auc = r.roc_auc;
    history[e].auc_value = aucsum[e] / (double)K;
  }
  return SRS_OK;
}

int srs_trainer_get_weights(const srs_trainer* t, const char* name, float* dst) {
  if (!t || !name || !dst) return failf(SRS_ERR_INVALID, "null argument");
  const Placed* x = nullptr;
  for (const Placed& y : t->place)
    if (y.name == name) x = &y;
  if (!x) return failf(SRS_ERR_MISSING, "the trainer has no tensor '%s'", name);
  CUDA_TRY(cudaSetDevice(t->device));
  CUDA_TRY(cudaStreamSynchronize(t->stream));
  if (x->table_row >= 0) {
    CUDA_TRY(cudaMemcpy2D(dst, (size_t)x->cols * sizeof(float), t->tab[0] + x->table_row * t->EP,
                           (size_t)t->EP * sizeof(float), (size_t)x->cols * sizeof(float), (size_t)x->rows,
                           cudaMemcpyDeviceToHost));
    return SRS_OK;
  }
  std::vector<float> blob(t->blob_floats), onehot;
  CUDA_TRY(cudaMemcpy(blob.data(), t->blob[0], blob.size() * sizeof(float), cudaMemcpyDeviceToHost));
  if (std::any_of(x->blocks.begin(), x->blocks.end(), [](const Block& k) { return k.onehot; })) {
    onehot.resize(t->onehot);
    CUDA_TRY(cudaMemcpy(onehot.data(), t->fo[0], onehot.size() * sizeof(float), cudaMemcpyDeviceToHost));
  }
  gather(*x, blob.data(), onehot.data(), dst);
  return SRS_OK;
}

}  // extern "C"
