// ncf_train.cu - `model.fit` of NeuralCF (neural_cf_model_1, NeuralCF.py:74-91) on the device: the C ABI's
// srs_trainer (include/srs_ctr.h) and its kernels.  DESIGN.md section 4.8.
//
// One step of batch B_b (rows order[off .. off + B_b) of the uploaded dataset), five launches, no host sync:
//   ncf_train_step_kernel  forward (the arithmetic of ncf_kernel) and backward, one thread per row; the Dense
//                          gradients as per-CTA partials summed over the CTA's rows in row order; each row's two
//                          embedding gradients and table rows to a list
//   table_grad_kernel      the table gradient of each distinct id of the batch: its rows' gradients added in row
//                          order by the thread of its first row (TF's _deduplicate_indexed_slices), into G
//   table_adam_kernel      Keras's sparse Adam on EVERY row of both tables (decay m and v, add the batch's G, update
//                          w); clears G
//   dense_adam_kernel      the CTA partials summed in CTA order, then TF's ApplyAdam on the Dense weights; advances
//                          the device-resident iteration counter
//   metrics_update_kernel  the step's probs / logits / labels into the epoch's history (metrics.cu)
// No float atomics: every sum has a fixed order, so a fit is bitwise reproducible.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/srs_ctr.h"
#include "kernels.h"
#include "ncf_layers.cuh"

namespace srs {

namespace {

constexpr int kTrainRows = 64;        // rows (threads) per CTA of the step kernel
constexpr int kAdamThreads = 512;     // the one CTA of dense_adam_kernel

struct TrainLayout {                  // the NcfParams blob layout (build_ncf), offsets in floats
  int n_layers, blob_floats;
  int w_off[3], b_off[3], out_w, out_b;
};

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
// no earlier entry has it.  G is zero on entry (table_adam_kernel clears what it reads).
__global__ void table_grad_kernel(const int32_t* __restrict__ trow, const float* __restrict__ gemb, int n,
                                  int EP, float* __restrict__ G) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int t = trow[e];
  for (int j = 0; j < e; ++j)
    if (trow[j] == t) return;
  float* g = G + (size_t)t * EP;
  for (int j = e; j < n; ++j) {
    if (trow[j] != t) continue;
    for (int k = 0; k < EP; ++k) g[k] = __fadd_rn(g[k], gemb[(size_t)j * EP + k]);
  }
}

// Keras's _resource_apply_sparse on every element of both tables: m = b1 m + (1-b1) G, v = b2 v + (1-b2) G^2,
// w -= alpha m / (sqrt(v) + eps), each operation rounded on its own (no contraction)
__global__ void table_adam_kernel(float* __restrict__ w, float* __restrict__ m, float* __restrict__ v,
                                  float* __restrict__ G, int64_t n, AdamHp h, const long long* __restrict__ it) {
  const float alpha = adam_alpha(h, *it);
  const float c1 = 1.f - h.b1, c2 = 1.f - h.b2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float g = G[i];
    if (g != 0.f) G[i] = 0.f;
    const float mi = __fadd_rn(__fmul_rn(h.b1, m[i]), __fmul_rn(c1, g));
    const float vi = __fadd_rn(__fmul_rn(h.b2, v[i]), __fmul_rn(c2, __fmul_rn(g, g)));
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

struct EpochMetrics {                 // one epoch's history state (the layout of srs_metrics' state)
  MetricsCounters cnt;
  double loss;
  MetricsReduce red;
};

int failf(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  return set_last_error(code, buf);
}

#define TRAIN_TRY(expr)                                                                           \
  do {                                                                                            \
    cudaError_t e__ = (expr);                                                                     \
    if (e__ != cudaSuccess)                                                                       \
      return failf(SRS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, \
                   __LINE__);                                                                     \
  } while (0)

// device allocations of one scope, freed when it ends
struct DeviceScratch {
  std::vector<void*> ptrs;
  ~DeviceScratch() { for (void* p : ptrs) cudaFree(p); }
  template <class T>
  cudaError_t alloc(T** p, size_t count) {
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) ptrs.push_back(q);
    *p = static_cast<T*>(q);
    return e;
  }
};

}  // namespace
}  // namespace srs

using namespace srs;

struct srs_trainer {
  srs_spec spec{};
  int device = 0;
  int E = 0, EP = 0, HP = 0;
  TrainLayout ly{};
  AdamHp hp{};
  int64_t tab_floats = 0;             // (n_movies + n_users) * EP
  float* tab[4] = {};                 // w, m, v, G   [n_movies + n_users][EP], padding zero
  float* blob[3] = {};                // w, m, v      [blob_floats]
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
  cudaFree(t->d_it);
  if (t->stream) cudaStreamDestroy(t->stream);
  delete t;
}

const srs_tensor* find_tensor(const srs_tensor* ts, int n, const char* name, int64_t rows, int64_t cols, int* rc) {
  for (int i = 0; i < n; ++i) {
    if (!ts[i].name || strcmp(ts[i].name, name) != 0) continue;
    if (ts[i].rows != rows || ts[i].cols != cols) {
      *rc = failf(SRS_ERR_SHAPE, "weight '%s' has shape [%lld,%lld], expected [%lld,%lld]", name,
                  (long long)ts[i].rows, (long long)ts[i].cols, (long long)rows, (long long)cols);
      return nullptr;
    }
    if (!ts[i].data || ts[i].location != SRS_HOST) {
      *rc = failf(SRS_ERR_INVALID, "weight '%s' must be a non-null host tensor", name);
      return nullptr;
    }
    return &ts[i];
  }
  *rc = failf(SRS_ERR_MISSING, "missing weight tensor '%s'", name);
  return nullptr;
}

// the Keras shape of a trainer tensor: table (layer -1), Dense kernel / bias of layer l; false if unknown
bool tensor_shape(const srs_trainer* t, const char* name, int* layer, int* is_bias, int64_t* rows, int64_t* cols) {
  const srs_spec& s = t->spec;
  if (!strcmp(name, "movieId_embedding")) { *layer = -1; *is_bias = 0; *rows = s.n_movies; *cols = t->E; return true; }
  if (!strcmp(name, "userId_embedding")) { *layer = -1; *is_bias = 1; *rows = s.n_users; *cols = t->E; return true; }
  const int L = s.n_hidden;
  for (int l = 0; l <= L; ++l) {
    char k[32], b[32];
    snprintf(k, sizeof(k), "dense_%d/kernel", l);
    snprintf(b, sizeof(b), "dense_%d/bias", l);
    const int in = l == 0 ? 2 * t->E : s.hidden[l - 1], out = l == L ? 1 : s.hidden[l];
    if (!strcmp(name, k)) { *layer = l; *is_bias = 0; *rows = in; *cols = out; return true; }
    if (!strcmp(name, b)) { *layer = l; *is_bias = 1; *rows = out; *cols = 1; return true; }
  }
  return false;
}

// element (i, j) of a Dense tensor -> its blob offset (build_ncf's layout), -1 for none
int blob_index(const srs_trainer* t, int layer, int is_bias, int64_t i, int64_t j) {
  const int L = t->spec.n_hidden, E = t->E, EP = t->EP, HP = t->HP;
  if (layer == L) return is_bias ? t->ly.out_b : t->ly.out_w + (int)i;
  if (is_bias) return t->ly.b_off[layer] + (int)i;
  const int row = layer == 0 ? (i < E ? (int)i : EP + (int)(i - E)) : (int)i;
  return t->ly.w_off[layer] + row * HP + (int)j;
}

}  // namespace

extern "C" {

int srs_trainer_create(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                       const srs_adam* hp, srs_trainer** out) {
  if (!spec || !out) return failf(SRS_ERR_INVALID, "null argument");
  *out = nullptr;
  const srs_spec& s = *spec;
  if (s.kind != SRS_NEURALCF) return failf(SRS_ERR_INVALID, "fit is implemented for NeuralCF (neural_cf_model_1) only");
  if (s.emb_dim < 1 || s.emb_dim > 64) return failf(SRS_ERR_INVALID, "emb_dim must be in 1..64");
  if (s.n_movies < 1 || s.n_users < 1) return failf(SRS_ERR_INVALID, "empty vocabulary");
  if (s.n_hidden < 1 || s.n_hidden > 3) return failf(SRS_ERR_INVALID, "1..3 hidden layers supported");
  int hmax = 0;
  for (int i = 0; i < s.n_hidden; ++i) {
    if (s.hidden[i] < 1 || s.hidden[i] > 32) return failf(SRS_ERR_INVALID, "hidden widths must be in 1..32");
    hmax = std::max(hmax, s.hidden[i]);
  }
  AdamHp h{0.001f, 0.9f, 0.999f, 1e-7f};              // Keras's Adam defaults
  if (hp) h = AdamHp{hp->lr, hp->beta_1, hp->beta_2, hp->epsilon};
  if (!(h.lr > 0.f && h.lr < 1e30f) || !(h.b1 >= 0.f && h.b1 < 1.f) || !(h.b2 >= 0.f && h.b2 < 1.f) ||
      !(h.eps > 0.f && h.eps < 1e30f))
    return failf(SRS_ERR_INVALID, "Adam needs lr > 0, 0 <= beta_1, beta_2 < 1 and epsilon > 0");
  if (n_tensors < 0 || (n_tensors > 0 && !tensors)) return failf(SRS_ERR_INVALID, "null tensors");
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return failf(SRS_ERR_CUDA, "no CUDA device available (%s); this library has no CPU path", cudaGetErrorString(ce));
  if (device < 0 || device >= ndev) return failf(SRS_ERR_INVALID, "device %d out of range", device);

  srs_trainer* t = new srs_trainer();
  t->spec = s;
  t->device = device;
  t->hp = h;
  t->E = s.emb_dim;
  t->EP = s.emb_dim <= 12 ? 12 : s.emb_dim <= 16 ? 16 : s.emb_dim <= 32 ? 32 : 64;
  t->HP = hmax <= 16 ? 16 : 32;
  const int E = t->E, EP = t->EP, HP = t->HP, L = s.n_hidden;
  // the blob layout of build_ncf: kernels [2EP or HP][HP] and biases [HP] per hidden layer, then out [HP], [4]
  int off = 0;
  t->ly.n_layers = L;
  for (int l = 0; l < L; ++l) {
    t->ly.w_off[l] = off; off += (l == 0 ? 2 * EP : HP) * HP;
    t->ly.b_off[l] = off; off += HP;
  }
  t->ly.out_w = off; off += HP;
  t->ly.out_b = off; off += 4;
  t->ly.blob_floats = off;
  t->tab_floats = ((int64_t)s.n_movies + s.n_users) * EP;

  std::vector<float> blob(off, 0.f);
  std::vector<std::pair<const float*, int64_t>> tabs;      // host source, rows
  int rc = SRS_OK;
  for (int which = 0; which < 2 && rc == SRS_OK; ++which) {
    const char* name = which ? "userId_embedding" : "movieId_embedding";
    const srs_tensor* x = find_tensor(tensors, n_tensors, name, which ? s.n_users : s.n_movies, E, &rc);
    if (x) tabs.push_back({x->data, x->rows});
  }
  for (int l = 0; l <= L && rc == SRS_OK; ++l) {
    for (int is_bias = 0; is_bias < 2 && rc == SRS_OK; ++is_bias) {
      char name[32];
      snprintf(name, sizeof(name), is_bias ? "dense_%d/bias" : "dense_%d/kernel", l);
      int layer, b; int64_t rows, cols;
      tensor_shape(t, name, &layer, &b, &rows, &cols);
      const srs_tensor* x = find_tensor(tensors, n_tensors, name, rows, cols, &rc);
      if (!x) break;
      for (int64_t i = 0; i < rows; ++i)
        for (int64_t j = 0; j < cols; ++j) blob[blob_index(t, layer, b, i, j)] = x->data[i * cols + j];
    }
  }
  if (rc != SRS_OK) { delete t; return rc; }

  ce = cudaSetDevice(device);
  if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&t->stream, cudaStreamNonBlocking);
  for (int k = 0; k < 4 && ce == cudaSuccess; ++k) ce = cudaMalloc(&t->tab[k], t->tab_floats * sizeof(float));
  for (int k = 0; k < 3 && ce == cudaSuccess; ++k) ce = cudaMalloc(&t->blob[k], (size_t)off * sizeof(float));
  if (ce == cudaSuccess) ce = cudaMalloc(&t->d_it, sizeof(long long));
  for (int k = 0; k < 4 && ce == cudaSuccess; ++k) ce = cudaMemset(t->tab[k], 0, t->tab_floats * sizeof(float));
  for (int k = 1; k < 3 && ce == cudaSuccess; ++k) ce = cudaMemset(t->blob[k], 0, (size_t)off * sizeof(float));
  if (ce == cudaSuccess) ce = cudaMemset(t->d_it, 0, sizeof(long long));
  if (ce == cudaSuccess) ce = cudaMemcpy(t->blob[0], blob.data(), (size_t)off * sizeof(float), cudaMemcpyHostToDevice);
  int64_t row0 = 0;
  for (size_t k = 0; k < tabs.size() && ce == cudaSuccess; ++k) {   // [V][E] -> [V][EP], padding stays zero
    ce = cudaMemcpy2D(t->tab[0] + row0 * EP, (size_t)EP * sizeof(float), tabs[k].first, (size_t)E * sizeof(float),
                      (size_t)E * sizeof(float), (size_t)tabs[k].second, cudaMemcpyHostToDevice);
    row0 += tabs[k].second;
  }
  if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
  if (ce != cudaSuccess) {
    trainer_free(t);
    return failf(ce == cudaErrorMemoryAllocation ? SRS_ERR_NOMEM : SRS_ERR_CUDA, "trainer setup failed: %s",
                 cudaGetErrorString(ce));
  }
  *out = t;
  return SRS_OK;
}

void srs_trainer_destroy(srs_trainer* t) { trainer_free(t); }

int64_t srs_trainer_iterations(const srs_trainer* t) { return t ? t->iterations : 0; }

int srs_trainer_fit_host(srs_trainer* t, const srs_batch* batch, const int32_t* labels, const int32_t* order,
                         int32_t batch_size, int32_t epochs, srs_eval_result* history) {
  if (!t || !batch || !labels || !order) return failf(SRS_ERR_INVALID, "null argument");
  const int n = batch->B;
  if (n < 1) return failf(SRS_ERR_INVALID, "fit needs at least one row");
  if (batch_size < 1) return failf(SRS_ERR_INVALID, "batch_size must be at least 1");
  if (epochs < 1) return failf(SRS_ERR_INVALID, "epochs must be at least 1");
  if (!batch->movie_id || !batch->user_id) return failf(SRS_ERR_INVALID, "movie_id and user_id are required");
  // every check before the first launch: a rejected call leaves the trainer as it was
  for (int i = 0; i < n; ++i)
    if (labels[i] != 0 && labels[i] != 1) return failf(SRS_ERR_INVALID, "label of row %d is %d, not 0 or 1", i, labels[i]);
  for (int i = 0; i < n; ++i) {
    if ((unsigned)batch->movie_id[i] >= (unsigned)t->spec.n_movies)
      return failf(SRS_ERR_RANGE, "movieId %d of row %d is outside [0, %d)", batch->movie_id[i], i, t->spec.n_movies);
    if ((unsigned)batch->user_id[i] >= (unsigned)t->spec.n_users)
      return failf(SRS_ERR_RANGE, "userId %d of row %d is outside [0, %d)", batch->user_id[i], i, t->spec.n_users);
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
  TRAIN_TRY(cudaSetDevice(t->device));
  const int EP = t->EP, Bmax = std::min(batch_size, n);
  const int n_cta = (Bmax + kTrainRows - 1) / kTrainRows;
  cudaStream_t s = t->stream;
  DeviceScratch sc;
  int32_t *d_movie, *d_user, *d_label, *d_order, *d_lab_b, *d_trow;
  float *d_probs, *d_logits, *d_gemb, *d_part;
  EpochMetrics* d_met;
  TRAIN_TRY(sc.alloc(&d_movie, n));
  TRAIN_TRY(sc.alloc(&d_user, n));
  TRAIN_TRY(sc.alloc(&d_label, n));
  TRAIN_TRY(sc.alloc(&d_order, (size_t)epochs * n));
  TRAIN_TRY(sc.alloc(&d_lab_b, Bmax));
  TRAIN_TRY(sc.alloc(&d_trow, 2 * (size_t)Bmax));
  TRAIN_TRY(sc.alloc(&d_probs, Bmax));
  TRAIN_TRY(sc.alloc(&d_logits, Bmax));
  TRAIN_TRY(sc.alloc(&d_gemb, 2 * (size_t)Bmax * EP));
  TRAIN_TRY(sc.alloc(&d_part, (size_t)n_cta * t->ly.blob_floats));
  TRAIN_TRY(sc.alloc(&d_met, epochs));
  TRAIN_TRY(cudaMemcpyAsync(d_movie, batch->movie_id, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  TRAIN_TRY(cudaMemcpyAsync(d_user, batch->user_id, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  TRAIN_TRY(cudaMemcpyAsync(d_label, labels, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  TRAIN_TRY(cudaMemcpyAsync(d_order, order, (size_t)epochs * n * 4, cudaMemcpyHostToDevice, s));
  TRAIN_TRY(cudaMemsetAsync(d_met, 0, sizeof(EpochMetrics) * epochs, s));

  int dev_sms = 132;
  cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, t->device);
  const int adam_blocks = (int)std::min<int64_t>((t->tab_floats + 255) / 256, (int64_t)dev_sms * 8);
  StepArgs a{};
  a.tab = t->tab[0]; a.blob = t->blob[0];
  a.movie = d_movie; a.user = d_user; a.label = d_label;
  a.n_movies = t->spec.n_movies;
  a.probs = d_probs; a.logits = d_logits; a.labels = d_lab_b; a.trow = d_trow; a.gemb = d_gemb; a.part = d_part;
  int64_t steps = 0;
  for (int e = 0; e < epochs; ++e) {
    for (int off = 0; off < n; off += batch_size) {
      a.B = std::min(batch_size, n - off);
      a.order = d_order + (size_t)e * n + off;
      TRAIN_TRY(launch_step(EP, t->HP, a, t->ly, s));
      table_grad_kernel<<<(2 * a.B + 127) / 128, 128, 0, s>>>(d_trow, d_gemb, 2 * a.B, EP, t->tab[3]);
      table_adam_kernel<<<adam_blocks, 256, 0, s>>>(t->tab[0], t->tab[1], t->tab[2], t->tab[3], t->tab_floats, t->hp,
                                                   t->d_it);
      dense_adam_kernel<<<1, kAdamThreads, 0, s>>>(d_part, (a.B + kTrainRows - 1) / kTrainRows, t->ly.blob_floats,
                                                   t->blob[0], t->blob[1], t->blob[2], t->hp, t->d_it);
      g_launch_count += 3;
      TRAIN_TRY(cudaGetLastError());
      TRAIN_TRY(launch_metrics_update(d_probs, d_logits, d_lab_b, a.B, &d_met[e].cnt, &d_met[e].red, &d_met[e].loss, 1,
                                      s));
      ++steps;
    }
  }
  std::vector<EpochMetrics> met(epochs);
  TRAIN_TRY(cudaMemcpyAsync(met.data(), d_met, sizeof(EpochMetrics) * epochs, cudaMemcpyDeviceToHost, s));
  TRAIN_TRY(cudaStreamSynchronize(s));
  t->iterations += steps;
  for (int e = 0; e < epochs; ++e) {
    if (met[e].cnt.err) return failf(SRS_ERR_INVALID, "epoch %d produced a probability that is NaN or outside [0, 1]", e);
    if (history) metrics_summarise(met[e].cnt.hist, met[e].cnt.correct, met[e].loss, &history[e], nullptr);
  }
  return SRS_OK;
}

int srs_trainer_get_weights(const srs_trainer* t, const char* name, float* dst) {
  if (!t || !name || !dst) return failf(SRS_ERR_INVALID, "null argument");
  int layer, is_bias;
  int64_t rows, cols;
  if (!tensor_shape(t, name, &layer, &is_bias, &rows, &cols))
    return failf(SRS_ERR_MISSING, "the trainer has no tensor '%s'", name);
  TRAIN_TRY(cudaSetDevice(t->device));
  TRAIN_TRY(cudaStreamSynchronize(t->stream));
  if (layer < 0) {
    const int64_t row0 = is_bias ? t->spec.n_movies : 0;      // is_bias marks the user table here
    TRAIN_TRY(cudaMemcpy2D(dst, (size_t)cols * sizeof(float), t->tab[0] + row0 * t->EP, (size_t)t->EP * sizeof(float),
                           (size_t)cols * sizeof(float), (size_t)rows, cudaMemcpyDeviceToHost));
    return SRS_OK;
  }
  std::vector<float> blob(t->ly.blob_floats);
  TRAIN_TRY(cudaMemcpy(blob.data(), t->blob[0], blob.size() * sizeof(float), cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < rows; ++i)
    for (int64_t j = 0; j < cols; ++j) dst[i * cols + j] = blob[blob_index(t, layer, is_bias, i, j)];
  return SRS_OK;
}

}  // extern "C"
