// ncf_train.cu - the forward / backward step of NeuralCF's `model.fit` (neural_cf_model_1, NeuralCF.py:74-91);
// the trainer that drives it (dedupe, Adam, metrics) is srs_trainer in trainer.cu.  DESIGN.md section 4.8.
//
// ncf_train_step_kernel<EP, HP>: one thread per row, 64 rows per CTA.  The forward is ncf_kernel's arithmetic
// (ncf_layers.cuh); the backward keeps each row's x, every layer's output and delta and dL/dz in shared memory, writes
// the row's two embedding gradients and table rows to a list, and thread q sums Dense parameter q's gradient over
// the CTA's rows in row order into a per-CTA partial.  No float atomics.
#include <cuda_runtime.h>

#include "kernels.h"
#include "ncf_layers.cuh"

namespace srs {

namespace {

constexpr int kTrainRows = 64;        // rows (threads) per CTA of the step kernel

struct TrainLayout {                  // the step kernel's view of NcfParams' blob layout, offsets in floats
  int n_layers, blob_floats;
  int w_off[3], b_off[3], out_w, out_b;
};

TrainLayout train_layout(const NcfParams& p) {      // offsets past n_layers are zero, and not read
  return TrainLayout{p.n_layers, p.blob_floats, {p.w_off[0], p.w_off[1], p.w_off[2]},
                     {p.b_off[0], p.b_off[1], p.b_off[2]}, p.out_w, p.out_b};
}

template <int EP, int HP>
__global__ void __launch_bounds__(kTrainRows) ncf_train_step_kernel(NcfStepArgs a, TrainLayout ly) {
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
    const float w = a.weight ? __ldg(a.weight + row) : 1.f;   // the row's weight (1: unweighted)
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
    if (a.weight) a.weights[r] = w;
#pragma unroll
    for (int q = 0; q < EP / 4; ++q) {
      const float4 mv = ldg4(mrow + 4 * q), uv = ldg4(urow + 4 * q);
      rec[4 * q] = mv.x; rec[4 * q + 1] = mv.y; rec[4 * q + 2] = mv.z; rec[4 * q + 3] = mv.w;
      rec[EP + 4 * q] = uv.x; rec[EP + 4 * q + 1] = uv.y; rec[EP + 4 * q + 2] = uv.z; rec[EP + 4 * q + 3] = uv.w;
    }
    // backward: dL/dz = (w (p - y)) / B (w = 1 unweighted), relu' = [a > 0] = [h > 0]
    const float dz = row_dz(p, y, a.weight != nullptr, w, a.B);
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

int step_smem_bytes(int EP, int HP, int n_layers, int blob_floats) {
  return (blob_floats + kTrainRows * (2 * EP + 2 * n_layers * HP + 1)) * (int)sizeof(float);
}

template <int EP, int HP>
cudaError_t launch_step_t(const NcfStepArgs* a, const TrainLayout& ly, cudaStream_t s) {
  const int smem = step_smem_bytes(EP, HP, ly.n_layers, ly.blob_floats);
  if (!a)                                             // the opt-in on the current device, no launch
    return cudaFuncSetAttribute(ncf_train_step_kernel<EP, HP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  ncf_train_step_kernel<EP, HP><<<ncf_train_ctas(a->B), kTrainRows, smem, s>>>(*a, ly);
  ++g_launch_count;
  return cudaGetLastError();
}

}  // namespace

int ncf_train_ctas(int B) { return (B + kTrainRows - 1) / kTrainRows; }

cudaError_t launch_ncf_train_step(const NcfStepArgs* a, const NcfParams& p, cudaStream_t s) {
  TrainLayout ly = train_layout(p);
  if (!a) {                // the opt-in is at 3 hidden layers, the largest step: each hidden layer past p's adds a
    ly.blob_floats += (3 - ly.n_layers) * (p.HP * p.HP + p.HP);   // kernel [HP][HP] and a bias [HP] (place_ncf)
    ly.n_layers = 3;
  }
#define SRS_TRAIN_CASE(E_, H_) \
  if (p.EP == E_ && p.HP == H_) return launch_step_t<E_, H_>(a, ly, s);
  SRS_TRAIN_CASE(12, 16) SRS_TRAIN_CASE(16, 16) SRS_TRAIN_CASE(32, 16) SRS_TRAIN_CASE(64, 16)
  SRS_TRAIN_CASE(12, 32) SRS_TRAIN_CASE(16, 32) SRS_TRAIN_CASE(32, 32) SRS_TRAIN_CASE(64, 32)
#undef SRS_TRAIN_CASE
  return cudaErrorInvalidValue;
}

}  // namespace srs
