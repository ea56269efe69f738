// ncf_train.cu - `model.fit` on the device: the C ABI's srs_trainer (include/srs_ctr.h), which trains NeuralCF
// (neural_cf_model_1, NeuralCF.py:74-91; DESIGN.md section 4.8), DeepFM (DeepFM.py; section 4.9, its step kernel
// in deepfm_train.cu), Wide&Deep (WideNDeep.py; section 4.18, its step kernel in widendeep_train.cu) and DeepFM_v2
// (DeepFM_v2.py; section 4.19, its step kernel in deepfm2_train.cu) and DIEN (DIEN.py; section 4.20, its step kernel
// in dien_train.cu, its fit in srs_trainer_fit_dien_host), and the kernels the models share: dedupe, the two forms of
// Adam, metrics.
//
// NeuralCF's step of batch B_b (rows order[off .. off + B_b) of the uploaded dataset), five launches, no host sync:
//   ncf_train_step_kernel  forward (the arithmetic of ncf_kernel) and backward, one thread per row; the Dense
//                          gradients as per-CTA partials summed over the CTA's rows in row order; each row's two
//                          embedding gradients and table rows to a list
//   table_grad_kernel      the table gradient of each distinct id of the batch: its rows' gradients added in row
//                          order by the thread of its first row (TF's _deduplicate_indexed_slices), into G
//   table_adam_kernel<false>  Keras's sparse Adam on EVERY row of both tables (decay m and v, add the batch's G, update
//                          w); clears G
//   dense_adam_kernel      the CTA partials summed in CTA order, then TF's ApplyAdam on the Dense weights; advances
//                          the device-resident iteration counter
//   metrics_update_kernel  the step's probs / logits / labels into the epoch's history (metrics.cu)
// DeepFM's step is seven launches: deepfm_train_step_kernel, table_grad_kernel over its table entries and again over
// its one-hot entries, table_adam_kernel<false> over the six tables and <true> over dense_2/kernel's one-hot rows,
// dense_adam_kernel, metrics_update_kernel; plus deepfm_permute_kernel once per epoch.
// Wide&Deep's step is seven launches of the same shape: widendeep_train_step_kernel, table_grad_kernel over its ten
// tables' entries and again (width 1) over its wide entries, table_adam_kernel<false> over the ten tables and <true>
// over the cross_buckets wide rows of dense_2/kernel, dense_adam_kernel, metrics_update_kernel; plus
// widendeep_permute_kernel once per epoch.
// DeepFM_v2's step is seven launches of the same shape again: deepfm2_train_step_kernel, table_grad_kernel over its
// four tables' entries and (width 1) over its one-hot entries, table_adam_kernel<false> over the four tables and
// <true> over first_cat/kernel's one-hot rows, dense_adam_kernel, metrics_update_kernel; plus deepfm_permute_kernel
// (it reads DeepFM's columns) once per epoch.
// DIEN's step is six launches and no permute (the step kernel reads its rows through the order): dien_train_step_kernel,
// table_grad_kernel over its (2T + 3) B entries, table_adam_kernel<false> over its four tables, dense_adam_kernel,
// dien_final_loss_kernel (the batch's final_loss sum) and metrics_update_kernel (with the batch's own histogram);
// plus launch_auc_value once per epoch.
// No float atomics: every sum has a fixed order, so a fit is bitwise reproducible.
//
// Validation (srs_trainer_fit_validate_host) and srs_trainer_evaluate_host run the serving forward over the
// trainer's arrays (ncf_kernel, deepfm_kernel, embmlp_kernel, deepfm2_kernel) and one metrics_update_kernel over all the rows: two launches, with the
// bits of a CTRModel built from the exported weights.  The trainer's arrays hold the weights where the serving
// builders put them: both place them through placement.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"
#include "ncf_layers.cuh"
#include "placement.h"

namespace srs {

namespace {

constexpr int kTrainRows = 64;        // rows (threads) per CTA of the step kernel
constexpr int kAdamThreads = 512;     // the one CTA of dense_adam_kernel

struct TrainLayout {                  // the step kernel's view of NcfParams' blob layout, offsets in floats
  int n_layers, blob_floats;
  int w_off[3], b_off[3], out_w, out_b;
};

TrainLayout train_layout(const NcfParams& p) {
  TrainLayout ly{};
  ly.n_layers = p.n_layers;
  ly.blob_floats = p.blob_floats;
  for (int l = 0; l < p.n_layers; ++l) { ly.w_off[l] = p.w_off[l]; ly.b_off[l] = p.b_off[l]; }
  ly.out_w = p.out_w;
  ly.out_b = p.out_b;
  return ly;
}

struct StepArgs {
  const float* tab;                   // [n_movies + n_users][EP]: movie rows, then user rows
  const float* blob;                  // Dense weights
  const int32_t* movie;               // the dataset [n]
  const int32_t* user;
  const int32_t* label;
  const int32_t* order;               // this step's rows [B]
  int B, n_movies;
  float* probs;                       // [B] outputs of the step, before its update
  float* logits;
  int32_t* labels;                    // [B] the step's labels, for the metrics
  int32_t* trow;                      // [2B] table row of each (movie, user) entry: movie r at r, user r at B + r
  float* gemb;                        // [2B][EP] the entries' embedding gradients
  float* part;                        // [gridDim.x][blob_floats] per-CTA Dense gradient sums
};

struct AdamHp { float lr, b1, b2, eps; };

// Keras's step size for t = iterations + 1 (float32): lr * sqrt(1 - beta_2^t) / (1 - beta_1^t)
__device__ __forceinline__ float adam_alpha(const AdamHp& h, long long it) {
  const float t = (float)(it + 1);
  return h.lr * (sqrtf(1.f - powf(h.b2, t)) / (1.f - powf(h.b1, t)));
}

template <int EP, int HP>
__global__ void __launch_bounds__(kTrainRows) ncf_train_step_kernel(StepArgs a, TrainLayout ly) {
  extern __shared__ __align__(16) float sw[];
  const int L = ly.n_layers;
  const int RS = 2 * EP + 2 * L * HP + 1;       // per row: x [2EP] | act l [HP] | delta l [HP] | dz
  float* srec = sw + ly.blob_floats;
  for (int i = threadIdx.x; i < ly.blob_floats; i += blockDim.x) sw[i] = __ldg(a.blob + i);
  __syncthreads();
  const int tid = threadIdx.x;
  const int r = blockIdx.x * kTrainRows + tid;
  float* rec = srec + tid * RS;
  float* act = rec + 2 * EP;
  float* dlt = act + L * HP;
  if (r < a.B) {
    const int row = __ldg(a.order + r);
    const int mid = __ldg(a.movie + row), uid = __ldg(a.user + row), y = __ldg(a.label + row);
    const float* mrow = a.tab + (size_t)mid * EP;
    const float* urow = a.tab + (size_t)(a.n_movies + uid) * EP;
    // forward: ncf_kernel's arithmetic for neural_cf_model_1
    float h[HP];
#pragma unroll
    for (int j = 0; j < HP; ++j) h[j] = sw[ly.b_off[0] + j];
    first_layer_accum<EP, HP>(h, mrow, sw + ly.w_off[0]);
    first_layer_accum<EP, HP>(h, urow, sw + ly.w_off[0] + EP * HP);
#pragma unroll
    for (int j = 0; j < HP; ++j) { h[j] = fmaxf(h[j], 0.f); act[j] = h[j]; }
    for (int l = 1; l < L; ++l) {
      hidden_layer<HP>(h, sw + ly.w_off[l], sw + ly.b_off[l]);
#pragma unroll
      for (int j = 0; j < HP; ++j) act[l * HP + j] = h[j];
    }
    float z = sw[ly.out_b];
#pragma unroll
    for (int j = 0; j < HP; ++j) z = fmaf(h[j], sw[ly.out_w + j], z);
    const float p = sigmoidf_acc(z);
    a.probs[r] = p;
    a.logits[r] = z;
    a.labels[r] = y;
#pragma unroll
    for (int q = 0; q < EP / 4; ++q) {
      const float4 mv = ldg4(mrow + 4 * q), uv = ldg4(urow + 4 * q);
      rec[4 * q] = mv.x; rec[4 * q + 1] = mv.y; rec[4 * q + 2] = mv.z; rec[4 * q + 3] = mv.w;
      rec[EP + 4 * q] = uv.x; rec[EP + 4 * q + 1] = uv.y; rec[EP + 4 * q + 2] = uv.z; rec[EP + 4 * q + 3] = uv.w;
    }
    // backward: dL/dz = (p - y) / B, relu' = [a > 0] = [h > 0]
    const float dz = (p - (float)y) / (float)a.B;
    rec[RS - 1] = dz;
    float d[HP];
#pragma unroll
    for (int j = 0; j < HP; ++j) d[j] = h[j] > 0.f ? dz * sw[ly.out_w + j] : 0.f;
    for (int l = L - 1; l >= 1; --l) {
#pragma unroll
      for (int j = 0; j < HP; ++j) dlt[l * HP + j] = d[j];
      float dn[HP];
      const float* W = sw + ly.w_off[l];
#pragma unroll
      for (int k = 0; k < HP; ++k) {
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < HP; ++j) s = fmaf(W[k * HP + j], d[j], s);
        dn[k] = act[(l - 1) * HP + k] > 0.f ? s : 0.f;
      }
#pragma unroll
      for (int k = 0; k < HP; ++k) d[k] = dn[k];
    }
#pragma unroll
    for (int j = 0; j < HP; ++j) dlt[j] = d[j];
    // the two embedding rows' gradients: x-gradient = W0 . delta_0
    const float* W0 = sw + ly.w_off[0];
#pragma unroll 4
    for (int k = 0; k < 2 * EP; ++k) {
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < HP; ++j) s = fmaf(W0[k * HP + j], d[j], s);
      const int e = k < EP ? r : a.B + r;
      a.gemb[(size_t)e * EP + (k % EP)] = s;
    }
    a.trow[r] = mid;
    a.trow[a.B + r] = a.n_movies + uid;
  }
  __syncthreads();
  // Dense gradients of this CTA's rows: parameter q = sum over rows in row order of (input . delta)
  const int nv = min(kTrainRows, a.B - (int)blockIdx.x * kTrainRows);
  const int dz_off = RS - 1;
  for (int q = tid; q < ly.blob_floats; q += kTrainRows) {
    int ao = -2, bo = 0;                               // ao: -2 zero (padding), -1 the constant 1
    for (int l = 0; l < L; ++l) {
      const int K = l == 0 ? 2 * EP : HP;
      if (q >= ly.w_off[l] && q < ly.w_off[l] + K * HP) {
        const int k = (q - ly.w_off[l]) / HP, j = (q - ly.w_off[l]) % HP;
        ao = l == 0 ? k : 2 * EP + (l - 1) * HP + k;
        bo = 2 * EP + L * HP + l * HP + j;
      } else if (q >= ly.b_off[l] && q < ly.b_off[l] + HP) {
        ao = -1;
        bo = 2 * EP + L * HP + l * HP + (q - ly.b_off[l]);
      }
    }
    if (q >= ly.out_w && q < ly.out_w + HP) { ao = 2 * EP + (L - 1) * HP + (q - ly.out_w); bo = dz_off; }
    if (q == ly.out_b) { ao = -1; bo = dz_off; }
    float s = 0.f;
    if (ao >= 0) {
      for (int i = 0; i < nv; ++i) s = fmaf(srec[i * RS + ao], srec[i * RS + bo], s);
    } else if (ao == -1) {
      for (int i = 0; i < nv; ++i) s += srec[i * RS + bo];
    }
    a.part[(size_t)blockIdx.x * ly.blob_floats + q] = s;
  }
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
// kApplyAdam = true, ApplyAdam's dense form (DeepFM's one-hot rows of dense_2/kernel): m += (G - m)(1-b1),
// v += (G^2 - v)(1-b2).  Then w -= alpha m / (sqrt(v) + eps).  Each operation is rounded on its own (no contraction).
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

int step_smem_bytes(int EP, int HP, const TrainLayout& ly) {
  return (ly.blob_floats + kTrainRows * (2 * EP + 2 * ly.n_layers * HP + 1)) * (int)sizeof(float);
}

template <int EP, int HP>
cudaError_t launch_step_t(const StepArgs& a, const TrainLayout& ly, cudaStream_t s) {
  const int smem = step_smem_bytes(EP, HP, ly);
  static int attr_set = 0;                              // the largest size opted in so far
  if (smem > 48 * 1024 && smem > attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(ncf_train_step_kernel<EP, HP>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    attr_set = smem;
  }
  ncf_train_step_kernel<EP, HP><<<(a.B + kTrainRows - 1) / kTrainRows, kTrainRows, smem, s>>>(a, ly);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_step(int EP, int HP, const StepArgs& a, const TrainLayout& ly, cudaStream_t s) {
#define SRS_TRAIN_CASE(E_, H_) \
  if (EP == E_ && HP == H_) return launch_step_t<E_, H_>(a, ly, s);
  SRS_TRAIN_CASE(12, 16) SRS_TRAIN_CASE(16, 16) SRS_TRAIN_CASE(32, 16) SRS_TRAIN_CASE(64, 16)
  SRS_TRAIN_CASE(12, 32) SRS_TRAIN_CASE(16, 32) SRS_TRAIN_CASE(32, 32) SRS_TRAIN_CASE(64, 32)
#undef SRS_TRAIN_CASE
  return cudaErrorInvalidValue;
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
  int64_t tab_floats = 0;             // (sum of the tables' rows) * EP
  float* tab[4] = {};                 // w, m, v, G   [rows][EP], padding zero
  float* blob[3] = {};                // w, m, v      [blob_floats]
  int64_t onehot = 0;                 // the one-hot rows: DeepFM's dense_2/kernel and DeepFM_v2's first_cat/kernel
                                      // (fm1_width), Wide&Deep's wide rows of dense_2/kernel
  float* fo[4] = {};                  // w, m, v, G   [onehot]
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

// a DeepFM (wd: Wide&Deep) dataset of n rows on the device
DeepFmRows deepfm_rows(Scratch& sc, int n, bool wd, cudaError_t* e) {
  DeepFmRows r{};
  *e = sc.alloc(&r.movie, n);
  if (*e == cudaSuccess && wd) *e = sc.alloc(&r.rated, n);
  if (*e == cudaSuccess) *e = sc.alloc(&r.user, n);
  if (*e == cudaSuccess) *e = sc.alloc(&r.mgenre, (size_t)n * 3);
  if (*e == cudaSuccess) *e = sc.alloc(&r.ugenre, (size_t)n * 5);
  if (*e == cudaSuccess) *e = sc.alloc(&r.numerics, (size_t)n * kNumNumerics);
  if (*e == cudaSuccess) *e = sc.alloc(&r.label, n);
  return r;
}

// The checks of rows the trainer reads (fit, validation, evaluate), all made before any launch.  `what` prefixes
// the messages: "" or "validation data: ".
int check_rows(const srs_trainer* t, const srs_batch* batch, const int32_t* labels, const char* what) {
  const bool fm = t->spec.kind == SRS_DEEPFM || t->spec.kind == SRS_DEEPFM_V2, wd = t->spec.kind == SRS_WIDENDEEP;
  const int n = batch->B;
  if (!batch->movie_id || !batch->user_id) return failf(SRS_ERR_INVALID, "%smovie_id and user_id are required", what);
  if (fm && (!batch->movie_genre || !batch->user_genre || !batch->numerics))
    return failf(SRS_ERR_INVALID, "%s%s needs movie_genre, user_genre and numerics", what,
                 t->spec.kind == SRS_DEEPFM ? "DeepFM" : "DeepFM_v2");
  if (wd && (!batch->movie_genre || !batch->user_genre || !batch->numerics || !batch->hist || batch->hist_stride < 1))
    return failf(SRS_ERR_INVALID, "%sWide&Deep needs movie_genre, user_genre, numerics and hist (userRatedMovie1)",
                 what);
  for (int i = 0; i < n; ++i)
    if (labels[i] != 0 && labels[i] != 1)
      return failf(SRS_ERR_INVALID, "%slabel of row %d is %d, not 0 or 1", what, i, labels[i]);
  for (int i = 0; i < n; ++i) {
    if ((unsigned)batch->movie_id[i] >= (unsigned)t->spec.n_movies)
      return failf(SRS_ERR_RANGE, "%smovieId %d of row %d is outside [0, %d)", what, batch->movie_id[i], i,
                   t->spec.n_movies);
    if ((unsigned)batch->user_id[i] >= (unsigned)t->spec.n_users)
      return failf(SRS_ERR_RANGE, "%suserId %d of row %d is outside [0, %d)", what, batch->user_id[i], i,
                   t->spec.n_users);
  }
  for (int i = 0; fm && i < n; ++i) {                  // a negative genre is missing (deepfm_kernel's genre_id)
    if (batch->movie_genre[(size_t)i * 3] >= t->spec.n_genres)
      return failf(SRS_ERR_RANGE, "%smovieGenre1 index %d of row %d is outside [0, %d)", what,
                   batch->movie_genre[(size_t)i * 3], i, t->spec.n_genres);
    if (batch->user_genre[(size_t)i * 5] >= t->spec.n_genres)
      return failf(SRS_ERR_RANGE, "%suserGenre1 index %d of row %d is outside [0, %d)", what,
                   batch->user_genre[(size_t)i * 5], i, t->spec.n_genres);
  }
  for (int i = 0; wd && i < n; ++i) {                  // every genre slot; a negative genre is missing
    for (int k = 0; k < 3; ++k)
      if (batch->movie_genre[(size_t)i * 3 + k] >= t->spec.n_genres)
        return failf(SRS_ERR_RANGE, "%smovieGenre%d index %d of row %d is outside [0, %d)", what, k + 1,
                     batch->movie_genre[(size_t)i * 3 + k], i, t->spec.n_genres);
    for (int k = 0; k < 5; ++k)
      if (batch->user_genre[(size_t)i * 5 + k] >= t->spec.n_genres)
        return failf(SRS_ERR_RANGE, "%suserGenre%d index %d of row %d is outside [0, %d)", what, k + 1,
                     batch->user_genre[(size_t)i * 5 + k], i, t->spec.n_genres);
    const int rated = batch->hist[(size_t)i * batch->hist_stride];
    if ((unsigned)rated >= (unsigned)t->spec.n_movies)
      return failf(SRS_ERR_RANGE, "%suserRatedMovie1 %d of row %d is outside [0, %d)", what, rated, i,
                   t->spec.n_movies);
  }
  return SRS_OK;
}

// batch->B rows on the device, uploaded on s: the columns the trainer's model reads (NeuralCF: movie and user only;
// DeepFM and DeepFM_v2: also the genres and numerics; Wide&Deep: also hist's column 0) and the labels
cudaError_t upload_rows(Scratch& sc, int kind, const srs_batch* b, const int32_t* labels, DeepFmRows* r,
                        cudaStream_t s) {
  const size_t n = (size_t)b->B;
  const bool wd = kind == SRS_WIDENDEEP, fm = kind == SRS_DEEPFM || kind == SRS_DEEPFM_V2 || wd;
  cudaError_t e;
  if (fm) {
    *r = deepfm_rows(sc, (int)n, wd, &e);
  } else {
    *r = DeepFmRows{};
    e = sc.alloc(&r->movie, n);
    if (e == cudaSuccess) e = sc.alloc(&r->user, n);
    if (e == cudaSuccess) e = sc.alloc(&r->label, n);
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(r->movie, b->movie_id, n * 4, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(r->user, b->user_id, n * 4, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(r->label, labels, n * 4, cudaMemcpyHostToDevice, s);
  if (fm && e == cudaSuccess) e = cudaMemcpyAsync(r->mgenre, b->movie_genre, n * 3 * 4, cudaMemcpyHostToDevice, s);
  if (fm && e == cudaSuccess) e = cudaMemcpyAsync(r->ugenre, b->user_genre, n * 5 * 4, cudaMemcpyHostToDevice, s);
  if (fm && e == cudaSuccess)
    e = cudaMemcpyAsync(r->numerics, b->numerics, n * kNumNumerics * 4, cudaMemcpyHostToDevice, s);
  if (wd && e == cudaSuccess)
    e = cudaMemcpy2DAsync(r->rated, 4, b->hist, (size_t)b->hist_stride * 4, 4, n, cudaMemcpyHostToDevice, s);
  return e;
}

// `model.evaluate` of the trainer's current weights over n device rows, two launches on s: the serving forward
// (ncf_kernel, deepfm_kernel, embmlp_kernel or deepfm2_kernel), then one metrics_update_kernel over all the rows into em.  `err` may
// be null for NeuralCF only (the genre checks of the others write it).
cudaError_t eval_rows(const srs_trainer* t, const DeepFmRows& r, int n, float* probs, float* logits, int* err,
                      MetricsState* em, cudaStream_t s) {
  BatchView b{};
  b.B = n;
  b.movie_id = r.movie; b.user_id = r.user;
  b.probs = probs; b.logits = logits; b.err_flag = err;
  cudaError_t e;
  if (t->spec.kind == SRS_DEEPFM) {
    b.movie_genre = r.mgenre; b.user_genre = r.ugenre; b.numerics = r.numerics;
    e = launch_deepfm(t->fm, b, s);
  } else if (t->spec.kind == SRS_WIDENDEEP) {
    b.movie_genre = r.mgenre; b.user_genre = r.ugenre; b.numerics = r.numerics;
    b.hist = r.rated; b.hist_stride = 1;
    e = launch_embmlp(t->emb, b, s);
  } else if (t->spec.kind == SRS_DEEPFM_V2) {
    b.movie_genre = r.mgenre; b.user_genre = r.ugenre; b.numerics = r.numerics;
    e = launch_deepfm2(t->fm2, b, s);
  } else {
    e = launch_ncf(t->ncf, b, s);
  }
  if (e != cudaSuccess) return e;
  return launch_metrics_update(probs, logits, r.label, n, &em->cnt, &em->red, &em->loss, 1, s);
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
  const bool fm = s.kind == SRS_DEEPFM, wd = s.kind == SRS_WIDENDEEP, fm2 = s.kind == SRS_DEEPFM_V2,
             dien = s.kind == SRS_DIEN;
  if (s.emb_dim < 1 || s.emb_dim > 64) return failf(SRS_ERR_INVALID, "emb_dim must be in 1..64");
  if (s.n_movies < 1 || s.n_users < 1) return failf(SRS_ERR_INVALID, "empty vocabulary");
  int hmax = 0;
  if (fm) {
    if (s.n_hidden != 2) return failf(SRS_ERR_INVALID, "DeepFM's fit needs exactly 2 hidden layers");
    if (s.n_genres < 1) return failf(SRS_ERR_INVALID, "empty genre vocabulary");
    for (int i = 0; i < 2; ++i)
      if (s.hidden[i] < 1 || s.hidden[i] > 64) return failf(SRS_ERR_INVALID, "DeepFM's hidden widths must be in 1..64");
  } else if (wd) {
    if (s.n_hidden != 2) return failf(SRS_ERR_INVALID, "Wide&Deep's fit needs exactly 2 hidden layers");
    if (s.n_genres < 1) return failf(SRS_ERR_INVALID, "empty genre vocabulary");
    if (s.cross_buckets < 1) return failf(SRS_ERR_INVALID, "Wide&Deep needs cross_buckets >= 1");
    for (int i = 0; i < 2; ++i)
      if (s.hidden[i] < 1 || s.hidden[i] > 128)
        return failf(SRS_ERR_INVALID, "Wide&Deep's hidden widths must be in 1..128");
  } else if (fm2) {
    if (s.n_hidden != 2) return failf(SRS_ERR_INVALID, "DeepFM_v2's fit needs exactly 2 hidden layers");
    if (s.proj_dim != 64) return failf(SRS_ERR_INVALID, "DeepFM_v2's fit needs proj_dim 64");
    if (s.n_genres < 1) return failf(SRS_ERR_INVALID, "empty genre vocabulary");
    if (s.hidden[0] < 1 || s.hidden[0] > 32 || s.hidden[1] < 1 || s.hidden[1] > 16)
      return failf(SRS_ERR_INVALID, "DeepFM_v2's hidden widths must be in 1..32 and 1..16");
  } else if (dien) {
    if (s.emb_dim > 32) return failf(SRS_ERR_INVALID, "DIEN's fit needs emb_dim in 1..32");
    if (s.hist_len < 1 || s.hist_len > kDienMaxT)
      return failf(SRS_ERR_INVALID, "DIEN's fit needs hist_len in 1..%d", kDienMaxT);
    if (s.au_hidden != 32) return failf(SRS_ERR_INVALID, "DIEN's fit needs au_hidden 32");
    if (s.n_hidden != 2) return failf(SRS_ERR_INVALID, "DIEN's fit needs exactly 2 hidden layers");
    if (s.n_genres < 1) return failf(SRS_ERR_INVALID, "empty genre vocabulary");
    if (s.hidden[0] < 1 || s.hidden[0] > 128 || s.hidden[1] < 1 || s.hidden[1] > 64)
      return failf(SRS_ERR_INVALID, "DIEN's hidden widths must be in 1..128 and 1..64");
  } else {
    if (s.n_hidden < 1 || s.n_hidden > 3) return failf(SRS_ERR_INVALID, "1..3 hidden layers supported");
    for (int i = 0; i < s.n_hidden; ++i) {
      if (s.hidden[i] < 1 || s.hidden[i] > 32) return failf(SRS_ERR_INVALID, "hidden widths must be in 1..32");
      hmax = std::max(hmax, s.hidden[i]);
    }
  }
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
  if (fm) {
    t->HP = 64;
    t->place = place_deepfm(s, EP, &t->fm);
    t->blob_floats = DeepFmBlob::of(EP).floats;
    t->onehot = (int64_t)2 * s.n_genres + s.n_movies + s.n_users;
  } else if (wd) {
    t->HP = 128;
    t->place = place_embmlp(s, EP, &t->emb);
    t->blob_floats = EmbMlpBlob::of(EP).floats;
    t->onehot = s.cross_buckets;
  } else if (fm2) {
    t->place = place_deepfm2(s, EP, &t->fm2);
    t->blob_floats = DeepFm2Blob::of(EP).floats;
    t->onehot = (int64_t)2 * s.n_genres + s.n_movies + s.n_users;
  } else if (dien) {
    t->place = place_dien(s, EP, true, &t->dien);   // the auxiliary head is part of the objective
    t->blob_floats = DienLayout::of(EP).floats;
  } else {
    t->HP = hmax <= 16 ? 16 : 32;
    t->place = place_ncf(s, EP, t->HP, &t->ncf);
    t->blob_floats = t->ncf.blob_floats;
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

  cudaError_t ce = cudaSetDevice(device);
  if (ce == cudaSuccess && (fm || fm2)) ce = setup_deepfm_attributes();   // validation and evaluate run deepfm_kernel
                                                                          //   (DeepFM_v2: deepfm2_kernel)
  if (ce == cudaSuccess && wd) ce = setup_embmlp_attributes();   //   (Wide&Deep: embmlp_kernel)
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
  // the serving parameters over the trainer's arrays
  auto table = [&](int k) { return t->tab[0] + t->place[k].table_row * EP; };
  if (fm) {
    t->fm.fm_movie = table(0); t->fm.fm_user = table(1); t->fm.fm_mgenre = table(2); t->fm.fm_ugenre = table(3);
    t->fm.deep_movie = table(4); t->fm.deep_user = table(5);
    point_into_blob(&t->fm, t->blob[0]);
    t->fm.first = t->fo[0];
  } else if (wd) {
    const float* tables[kWideDeepTables];
    for (int k = 0; k < kWideDeepTables; ++k) tables[k] = table(k);
    point_into_blob(&t->emb, tables, t->blob[0]);
    t->emb.wide = t->fo[0];
  } else if (fm2) {
    const float* tables[kDeepFm2Tables];
    for (int k = 0; k < kDeepFm2Tables; ++k) tables[k] = table(k);
    point_into_blob(&t->fm2, tables, t->blob[0]);
    t->fm2.first = t->fo[0];
  } else if (dien) {
    const float* tables[kDienTables];
    for (int k = 0; k < kDienTables; ++k) tables[k] = table(k);
    point_into_blob(&t->dien, tables, t->blob[0], blob.data());   // the step kernel reads b3 from the blob
  } else {
    t->ncf.movie = table(0);
    t->ncf.user = table(1);
    t->ncf.blob = t->blob[0];
  }
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
  if (k != SRS_NEURALCF && k != SRS_DEEPFM && k != SRS_WIDENDEEP && k != SRS_DEEPFM_V2 && k != SRS_DIEN)
    return failf(SRS_ERR_INVALID, "fit is implemented for NeuralCF (neural_cf_model_1), DeepFM, Wide&Deep, "
                 "DeepFM_v2 and DIEN only");
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
  if (!t || !batch || !labels || !order) return failf(SRS_ERR_INVALID, "null argument");
  if (t->spec.kind == SRS_DIEN) return dien_rejected("fit");
  const bool fm = t->spec.kind == SRS_DEEPFM, wd = t->spec.kind == SRS_WIDENDEEP, fm2 = t->spec.kind == SRS_DEEPFM_V2;
  const int n = batch->B;
  if (n < 1) return failf(SRS_ERR_INVALID, "fit needs at least one row");
  if (batch_size < 1) return failf(SRS_ERR_INVALID, "batch_size must be at least 1");
  if (epochs < 1) return failf(SRS_ERR_INVALID, "epochs must be at least 1");
  // every check before the first launch: a rejected call leaves the trainer as it was
  int rc = check_rows(t, batch, labels, "");
  if (rc != SRS_OK) return rc;
  {
    std::vector<char> seen(n);
    for (int e = 0; e < epochs; ++e) {
      std::fill(seen.begin(), seen.end(), 0);
      for (int i = 0; i < n; ++i) {
        const int r = order[(size_t)e * n + i];
        if (r < 0 || r >= n || seen[r]) return failf(SRS_ERR_INVALID, "order of epoch %d is not a permutation of 0..%d", e, n - 1);
        seen[r] = 1;
      }
    }
  }
  const int nv = val_batch ? val_batch->B : 0;         // validation rows; 0: no validation
  if (val_batch) {
    if (!val_labels) return failf(SRS_ERR_INVALID, "validation data: null labels");
    if (nv < 1) return failf(SRS_ERR_INVALID, "validation data: needs at least one row");
    if (val_freq < 1) return failf(SRS_ERR_INVALID, "validation_freq must be at least 1");
    rc = check_rows(t, val_batch, val_labels, "validation data: ");
    if (rc != SRS_OK) return rc;
  }
  CUDA_TRY(cudaSetDevice(t->device));
  const int EP = t->EP, Bmax = std::min(batch_size, n);
  const int n_ent = fm ? kDeepFmTables : wd ? kWideDeepTables : fm2 ? kDeepFm2Tables : 2;   // table entries per row
  auto step_ctas = [&](int B) {
    return fm ? deepfm_train_ctas(B) : wd ? widendeep_train_ctas(B) : fm2 ? deepfm2_train_ctas(B)
                                                                         : (B + kTrainRows - 1) / kTrainRows;
  };
  const int n_cta = step_ctas(Bmax);
  cudaStream_t s = t->stream;
  Scratch sc;
  int32_t *d_order, *d_trow, *d_lab_b = nullptr, *d_frow = nullptr;
  float *d_probs, *d_logits, *d_gemb, *d_part, *d_fgrad = nullptr;
  int* d_err = nullptr;
  MetricsState* d_met;
  CUDA_TRY(sc.alloc(&d_order, (size_t)epochs * n));
  CUDA_TRY(sc.alloc(&d_trow, (size_t)n_ent * Bmax));
  CUDA_TRY(sc.alloc(&d_probs, Bmax));
  CUDA_TRY(sc.alloc(&d_logits, Bmax));
  CUDA_TRY(sc.alloc(&d_gemb, (size_t)n_ent * Bmax * EP));
  CUDA_TRY(sc.alloc(&d_part, (size_t)n_cta * t->blob_floats));
  CUDA_TRY(sc.alloc(&d_met, epochs));
  CUDA_TRY(cudaMemcpyAsync(d_order, order, (size_t)epochs * n * 4, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemsetAsync(d_met, 0, sizeof(MetricsState) * epochs, s));
  DeepFmRows src{}, rows{};                            // the dataset, and (but NeuralCF) the epoch's rows in order
  CUDA_TRY(upload_rows(sc, t->spec.kind, batch, labels, &src, s));
  const int n_fent = wd ? 1 : 4;                       // one-hot entries per row (DeepFM, DeepFM_v2, Wide&Deep)
  if (fm || wd || fm2) {
    cudaError_t e;
    rows = deepfm_rows(sc, n, wd, &e);
    CUDA_TRY(e);
    CUDA_TRY(sc.alloc(&d_frow, n_fent * (size_t)Bmax));
    CUDA_TRY(sc.alloc(&d_fgrad, n_fent * (size_t)Bmax));
    CUDA_TRY(sc.alloc(&d_err, 1));
    CUDA_TRY(cudaMemsetAsync(d_err, 0, sizeof(int), s));
  } else {
    CUDA_TRY(sc.alloc(&d_lab_b, Bmax));
  }
  // validation: its rows uploaded once, in file order; each validated epoch's metrics in its own state
  DeepFmRows vrows{};
  float *d_vprobs = nullptr, *d_vlogits = nullptr;
  MetricsState* d_vmet = nullptr;
  if (nv) {
    CUDA_TRY(upload_rows(sc, t->spec.kind, val_batch, val_labels, &vrows, s));
    CUDA_TRY(sc.alloc(&d_vprobs, nv));
    CUDA_TRY(sc.alloc(&d_vlogits, nv));
    CUDA_TRY(sc.alloc(&d_vmet, epochs));
    CUDA_TRY(cudaMemsetAsync(d_vmet, 0, sizeof(MetricsState) * epochs, s));
  }

  int dev_sms = 132;
  cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, t->device);
  const int adam_blocks = (int)std::min<int64_t>((t->tab_floats + 255) / 256, (int64_t)dev_sms * 8);
  const int fo_blocks = (int)std::min<int64_t>((t->onehot + 255) / 256, (int64_t)dev_sms * 8);
  const TrainLayout ly = train_layout(t->ncf);
  StepArgs a{};
  a.tab = t->tab[0]; a.blob = t->blob[0];
  a.movie = src.movie; a.user = src.user; a.label = src.label;
  a.n_movies = t->spec.n_movies;
  a.probs = d_probs; a.logits = d_logits; a.labels = d_lab_b; a.trow = d_trow; a.gemb = d_gemb; a.part = d_part;
  DeepFmStepArgs f{};
  if (fm) {
    f.p = t->fm;
    for (int k = 0; k < kDeepFmTables; ++k) f.tab_row0[k] = t->place[k].table_row;   // the tables come first
    f.b.probs = d_probs; f.b.logits = d_logits; f.b.err_flag = d_err;
    f.trow = d_trow; f.gemb = d_gemb; f.frow = d_frow; f.fgrad = d_fgrad; f.part = d_part;
  }
  WideDeepStepArgs w{};
  if (wd) {
    w.p = t->emb;
    for (int k = 0; k < kWideDeepTables; ++k) w.tab_row0[k] = t->place[kEmbMlpSlotTable[k]].table_row;
    w.b.probs = d_probs; w.b.logits = d_logits; w.b.err_flag = d_err; w.b.hist_stride = 1;
    w.trow = d_trow; w.gemb = d_gemb; w.wrow = d_frow; w.wgrad = d_fgrad; w.part = d_part;
  }
  DeepFm2StepArgs v{};
  if (fm2) {
    v.p = t->fm2;
    for (int k = 0; k < kDeepFm2Tables; ++k) v.tab_row0[k] = t->place[k].table_row;   // the tables come first
    v.b.probs = d_probs; v.b.logits = d_logits; v.b.err_flag = d_err;
    v.trow = d_trow; v.gemb = d_gemb; v.frow = d_frow; v.fgrad = d_fgrad; v.part = d_part;
  }
  int64_t steps = 0;
  for (int e = 0; e < epochs; ++e) {
    if (fm || fm2) CUDA_TRY(launch_deepfm_permute(src, rows, d_order + (size_t)e * n, n, s));
    if (wd) CUDA_TRY(launch_widendeep_permute(src, rows, d_order + (size_t)e * n, n, s));
    for (int off = 0; off < n; off += batch_size) {
      const int B = std::min(batch_size, n - off);
      const int32_t* step_labels;
      if (fm || wd || fm2) {                           // the model's step, both dedupes, both forms of Adam
        BatchView& b = fm ? f.b : wd ? w.b : v.b;
        b.B = B;
        b.movie_id = rows.movie + off; b.user_id = rows.user + off;
        b.movie_genre = rows.mgenre + (size_t)off * 3; b.user_genre = rows.ugenre + (size_t)off * 5;
        b.numerics = rows.numerics + (size_t)off * kNumNumerics;
        if (wd) b.hist = rows.rated + off;
        step_labels = f.label = w.label = v.label = rows.label + off;
        CUDA_TRY(fm ? launch_deepfm_train_step(f, s) : wd ? launch_widendeep_train_step(w, s)
                                                          : launch_deepfm2_train_step(v, s));
        table_grad_kernel<<<(n_ent * B + 127) / 128, 128, 0, s>>>(d_trow, d_gemb, n_ent * B, EP, t->tab[3]);
        table_grad_kernel<<<(n_fent * B + 127) / 128, 128, 0, s>>>(d_frow, d_fgrad, n_fent * B, 1, t->fo[3]);
        table_adam_kernel<false><<<adam_blocks, 256, 0, s>>>(t->tab[0], t->tab[1], t->tab[2], t->tab[3],
                                                             t->tab_floats, t->hp, t->d_it);
        table_adam_kernel<true><<<fo_blocks, 256, 0, s>>>(t->fo[0], t->fo[1], t->fo[2], t->fo[3], t->onehot, t->hp,
                                                          t->d_it);
        dense_adam_kernel<<<1, kAdamThreads, 0, s>>>(d_part, step_ctas(B), t->blob_floats, t->blob[0],
                                                     t->blob[1], t->blob[2], t->hp, t->d_it);
        g_launch_count += 5;
      } else {
        a.B = B;
        a.order = d_order + (size_t)e * n + off;
        step_labels = d_lab_b;
        CUDA_TRY(launch_step(EP, t->HP, a, ly, s));
        table_grad_kernel<<<(2 * a.B + 127) / 128, 128, 0, s>>>(d_trow, d_gemb, 2 * a.B, EP, t->tab[3]);
        table_adam_kernel<false><<<adam_blocks, 256, 0, s>>>(t->tab[0], t->tab[1], t->tab[2], t->tab[3],
                                                             t->tab_floats, t->hp, t->d_it);
        dense_adam_kernel<<<1, kAdamThreads, 0, s>>>(d_part, (a.B + kTrainRows - 1) / kTrainRows, t->blob_floats,
                                                     t->blob[0], t->blob[1], t->blob[2], t->hp, t->d_it);
        g_launch_count += 3;
      }
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(launch_metrics_update(d_probs, d_logits, step_labels, B, &d_met[e].cnt, &d_met[e].red, &d_met[e].loss,
                                      1, s));
      ++steps;
    }
    // after the epoch's last update, on the same stream: no host synchronisation
    if (nv && (e + 1) % val_freq == 0) CUDA_TRY(eval_rows(t, vrows, nv, d_vprobs, d_vlogits, d_err, &d_vmet[e], s));
  }
  std::vector<MetricsState> met(epochs), vmet(nv ? epochs : 0);
  CUDA_TRY(cudaMemcpyAsync(met.data(), d_met, sizeof(MetricsState) * epochs, cudaMemcpyDeviceToHost, s));
  if (nv) CUDA_TRY(cudaMemcpyAsync(vmet.data(), d_vmet, sizeof(MetricsState) * epochs, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  t->iterations += steps;
  for (int e = 0; e < epochs; ++e) {
    const bool validated = nv && (e + 1) % val_freq == 0;
    if (met[e].cnt.err) return failf(SRS_ERR_INVALID, "epoch %d produced a probability that is NaN or outside [0, 1]", e);
    if (validated && vmet[e].cnt.err)
      return failf(SRS_ERR_INVALID, "the validation of epoch %d produced a probability that is NaN or outside [0, 1]",
                   e);
    if (history) metrics_summarise(met[e].cnt.hist, met[e].cnt.correct, met[e].loss, &history[e], nullptr);
    if (val_history) {
      val_history[e] = srs_eval_result{};
      if (validated) metrics_summarise(vmet[e].cnt.hist, vmet[e].cnt.correct, vmet[e].loss, &val_history[e], nullptr);
    }
  }
  return SRS_OK;
}

int srs_trainer_evaluate_host(srs_trainer* t, const srs_batch* batch, const int32_t* labels, srs_eval_result* out) {
  if (!t || !batch || !labels || !out) return failf(SRS_ERR_INVALID, "null argument");
  if (t->spec.kind == SRS_DIEN) return dien_rejected("evaluate");
  const int n = batch->B;
  if (n < 1) return failf(SRS_ERR_INVALID, "evaluate needs at least one row");
  const int rc = check_rows(t, batch, labels, "");
  if (rc != SRS_OK) return rc;
  CUDA_TRY(cudaSetDevice(t->device));
  cudaStream_t s = t->stream;
  Scratch sc;
  DeepFmRows rows{};
  float *d_probs, *d_logits;
  int* d_err;
  MetricsState* d_met;
  CUDA_TRY(upload_rows(sc, t->spec.kind, batch, labels, &rows, s));
  CUDA_TRY(sc.alloc(&d_probs, n));
  CUDA_TRY(sc.alloc(&d_logits, n));
  CUDA_TRY(sc.alloc(&d_err, 1));
  CUDA_TRY(sc.alloc(&d_met, 1));
  CUDA_TRY(cudaMemsetAsync(d_err, 0, sizeof(int), s));
  CUDA_TRY(cudaMemsetAsync(d_met, 0, sizeof(MetricsState), s));
  CUDA_TRY(eval_rows(t, rows, n, d_probs, d_logits, d_err, d_met, s));
  MetricsState met;
  CUDA_TRY(cudaMemcpyAsync(&met, d_met, sizeof(met), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  if (met.cnt.err) return failf(SRS_ERR_INVALID, "evaluate produced a probability that is NaN or outside [0, 1]");
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
  if (n < 1) return failf(SRS_ERR_INVALID, "fit needs at least one row");
  if (batch_size < 1) return failf(SRS_ERR_INVALID, "batch_size must be at least 1");
  if (epochs < 1) return failf(SRS_ERR_INVALID, "epochs must be at least 1");
  // every check before the first launch: a rejected call leaves the trainer as it was
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
  {
    std::vector<char> seen(n);
    for (int e = 0; e < epochs; ++e) {
      std::fill(seen.begin(), seen.end(), 0);
      for (int i = 0; i < n; ++i) {
        const int r = order[(size_t)e * n + i];
        if (r < 0 || r >= n || seen[r]) return failf(SRS_ERR_INVALID, "order of epoch %d is not a permutation of 0..%d", e, n - 1);
        seen[r] = 1;
      }
    }
  }
  CUDA_TRY(cudaSetDevice(t->device));
  const int EP = t->EP, Bmax = std::min(batch_size, n), K = (n + batch_size - 1) / batch_size;
  const int n_ent = 2 * T + 3;                          // table entries per row
  cudaStream_t s = t->stream;
  Scratch sc;
  int32_t *d_order, *d_movie, *d_user, *d_ug, *d_mg, *d_hist, *d_neg = nullptr, *d_label, *d_lab_b, *d_trow;
  float *d_num, *d_probs, *d_logits, *d_aux, *d_final, *d_gemb, *d_rec, *d_part;
  double *d_bloss, *d_auc, *d_aucsum;
  unsigned long long* d_bhist;
  MetricsState* d_met;
  const size_t N = (size_t)n;
  CUDA_TRY(sc.alloc(&d_order, (size_t)epochs * N));
  CUDA_TRY(sc.alloc(&d_movie, N));
  CUDA_TRY(sc.alloc(&d_user, N));
  CUDA_TRY(sc.alloc(&d_ug, N));
  CUDA_TRY(sc.alloc(&d_mg, N));
  CUDA_TRY(sc.alloc(&d_num, N * kNumNumerics));
  CUDA_TRY(sc.alloc(&d_hist, N * T));
  if (T > 1) CUDA_TRY(sc.alloc(&d_neg, N * (T - 1)));
  CUDA_TRY(sc.alloc(&d_label, N));
  CUDA_TRY(sc.alloc(&d_lab_b, Bmax));
  CUDA_TRY(sc.alloc(&d_probs, Bmax));
  CUDA_TRY(sc.alloc(&d_logits, Bmax));
  CUDA_TRY(sc.alloc(&d_aux, Bmax));
  CUDA_TRY(sc.alloc(&d_final, Bmax));
  CUDA_TRY(sc.alloc(&d_trow, (size_t)n_ent * Bmax));
  CUDA_TRY(sc.alloc(&d_gemb, (size_t)n_ent * Bmax * EP));
  CUDA_TRY(sc.alloc(&d_rec, dien_train_rec_floats(Bmax, T)));
  CUDA_TRY(sc.alloc(&d_part, (size_t)dien_train_ctas(Bmax) * t->blob_floats));
  CUDA_TRY(sc.alloc(&d_bloss, (size_t)epochs * K));
  CUDA_TRY(sc.alloc(&d_auc, (size_t)K));
  CUDA_TRY(sc.alloc(&d_aucsum, (size_t)epochs));
  CUDA_TRY(sc.alloc(&d_bhist, (size_t)K * 2 * kMetBins));
  CUDA_TRY(sc.alloc(&d_met, epochs));
  CUDA_TRY(cudaMemcpyAsync(d_order, order, (size_t)epochs * N * 4, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_movie, batch->movie_id, N * 4, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_user, batch->user_id, N * 4, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpy2DAsync(d_ug, 4, batch->user_genre, 5 * 4, 4, N, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpy2DAsync(d_mg, 4, batch->movie_genre, 3 * 4, 4, N, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_num, batch->numerics, N * kNumNumerics * 4, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpy2DAsync(d_hist, (size_t)T * 4, batch->hist, (size_t)batch->hist_stride * 4, (size_t)T * 4, N,
                             cudaMemcpyHostToDevice, s));
  if (T > 1)
    CUDA_TRY(cudaMemcpy2DAsync(d_neg, (size_t)(T - 1) * 4, neg_hist, (size_t)neg_stride * 4, (size_t)(T - 1) * 4, N,
                               cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_label, labels, N * 4, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemsetAsync(d_met, 0, sizeof(MetricsState) * epochs, s));

  int dev_sms = 132;
  cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, t->device);
  const int adam_blocks = (int)std::min<int64_t>((t->tab_floats + 255) / 256, (int64_t)dev_sms * 8);
  DienStepArgs a{};
  a.p = t->dien;
  a.blob = t->blob[0];
  a.movie = d_movie; a.user = d_user; a.ugenre = d_ug; a.mgenre = d_mg; a.numerics = d_num;
  a.hist = d_hist; a.neg = d_neg; a.label = d_label;
  for (int k = 0; k < kDienTables; ++k) a.tab_row0[k] = t->place[k].table_row;   // the tables come first
  a.probs = d_probs; a.logits = d_logits; a.aux = d_aux; a.labels = d_lab_b;
  a.trow = d_trow; a.gemb = d_gemb; a.rec = d_rec; a.part = d_part;
  for (int e = 0; e < epochs; ++e) {
    CUDA_TRY(cudaMemsetAsync(d_bhist, 0, (size_t)K * 2 * kMetBins * sizeof(unsigned long long), s));
    for (int k = 0; k < K; ++k) {
      const int off = k * batch_size, B = std::min(batch_size, n - off);
      a.B = B;
      a.order = d_order + (size_t)e * n + off;
      CUDA_TRY(launch_dien_train_step(a, s));
      table_grad_kernel<<<(n_ent * B + 127) / 128, 128, 0, s>>>(d_trow, d_gemb, n_ent * B, EP, t->tab[3]);
      table_adam_kernel<false><<<adam_blocks, 256, 0, s>>>(t->tab[0], t->tab[1], t->tab[2], t->tab[3],
                                                           t->tab_floats, t->hp, t->d_it);
      dense_adam_kernel<<<1, kAdamThreads, 0, s>>>(d_part, dien_train_ctas(B), t->blob_floats, t->blob[0],
                                                   t->blob[1], t->blob[2], t->hp, t->d_it);
      g_launch_count += 3;
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(launch_dien_final_loss(d_logits, d_lab_b, d_aux, B, d_final, d_bloss + (size_t)e * K + k, s));
      CUDA_TRY(launch_metrics_update(d_probs, d_logits, d_lab_b, B, &d_met[e].cnt, &d_met[e].red, nullptr, 0, s,
                                      d_bhist + (size_t)k * 2 * kMetBins));
    }
    CUDA_TRY(launch_auc_value(d_bhist, K, d_auc, d_aucsum + e, s));
  }
  std::vector<MetricsState> met(epochs);
  std::vector<double> bloss((size_t)epochs * K), aucsum(epochs);
  CUDA_TRY(cudaMemcpyAsync(met.data(), d_met, sizeof(MetricsState) * epochs, cudaMemcpyDeviceToHost, s));
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
