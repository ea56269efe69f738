// twotowers_train.cu - the forward / backward step of the two-tower model's `model.fit` (neural_cf_model_2 with its
// final Dense, NeuralCF.py:57-70); the trainer that drives it (dedupe, Adam, metrics) is srs_trainer in trainer.cu.
// DESIGN.md section 4.27.
//
// twotowers_train_step_kernel<EP, HP>: one thread per row, 64 rows per CTA, as ncf_train_step_kernel.  The forward is
// ncf_kernel's two-tower chain, op for op (ncf_layers.cuh), so a step's probabilities are the serving model's.  The
// backward keeps each row's two embedding rows, every layer's output and delta of both towers, the Dot d and dL/dz in
// shared memory, writes the row's two embedding gradients and table rows to a list, and thread q sums Dense parameter
// q's gradient over the CTA's rows in row order into a per-CTA partial.  No float atomics.
#include <cuda_runtime.h>

#include "kernels.h"
#include "ncf_layers.cuh"

namespace srs {

namespace {

constexpr int kTrainRows = 64;        // rows (threads) per CTA of the step kernel

struct TowerLayout {                  // the step kernel's view of NcfParams' two-tower blob layout, offsets in floats
  int n_layers, blob_floats;
  int w_off[6], b_off[6], out_w, out_b;   // item tower at [l], user tower at [3 + l]; past n_layers zero, not read
};

TowerLayout tower_layout(const NcfParams& p) {
  TowerLayout ly{p.n_layers, p.blob_floats, {}, {}, p.out_w, p.out_b};
  for (int i = 0; i < 6; ++i) { ly.w_off[i] = p.w_off[i]; ly.b_off[i] = p.b_off[i]; }
  return ly;
}

// per row, in floats: x [2EP] (item row, user row) | act [2][L][HP] | delta [2][L][HP] | d | dz
__host__ __device__ constexpr int row_floats(int EP, int HP, int L) { return 2 * EP + 4 * L * HP + 2; }

template <int EP, int HP>
__global__ void __launch_bounds__(kTrainRows) twotowers_train_step_kernel(NcfStepArgs a, TowerLayout ly) {
  extern __shared__ __align__(16) float sw[];
  const int L = ly.n_layers;
  const int RS = row_floats(EP, HP, L);
  const int ACT = 2 * EP, DLT = ACT + 2 * L * HP, D = DLT + 2 * L * HP, DZ = D + 1;
  float* srec = sw + ly.blob_floats;
  for (int i = threadIdx.x; i < ly.blob_floats; i += blockDim.x) sw[i] = __ldg(a.blob + i);
  __syncthreads();
  const int tid = threadIdx.x;
  const int r = blockIdx.x * kTrainRows + tid;
  float* rec = srec + tid * RS;
  if (r < a.B) {
    const int row = __ldg(a.order + r);
    const int mid = __ldg(a.movie + row), uid = __ldg(a.user + row), y = __ldg(a.label + row);
    const float w = a.weight ? __ldg(a.weight + row) : 1.f;   // the row's weight (1: unweighted)
    const float* mrow = a.tab + (size_t)mid * EP;
    const float* urow = a.tab + (size_t)(a.n_movies + uid) * EP;
    float* act_i = rec + ACT;
    float* act_u = act_i + L * HP;
    // forward: ncf_kernel's two-tower chain
    float hi[HP], hu[HP];
#pragma unroll
    for (int j = 0; j < HP; ++j) { hi[j] = sw[ly.b_off[0] + j]; hu[j] = sw[ly.b_off[3] + j]; }
    first_layer_accum<EP, HP>(hi, mrow, sw + ly.w_off[0]);
    first_layer_accum<EP, HP>(hu, urow, sw + ly.w_off[3]);
#pragma unroll
    for (int j = 0; j < HP; ++j) {
      hi[j] = fmaxf(hi[j], 0.f); hu[j] = fmaxf(hu[j], 0.f);
      act_i[j] = hi[j]; act_u[j] = hu[j];
    }
    for (int l = 1; l < L; ++l) {
      hidden_layer<HP>(hi, sw + ly.w_off[l], sw + ly.b_off[l]);
      hidden_layer<HP>(hu, sw + ly.w_off[3 + l], sw + ly.b_off[3 + l]);
#pragma unroll
      for (int j = 0; j < HP; ++j) { act_i[l * HP + j] = hi[j]; act_u[l * HP + j] = hu[j]; }
    }
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < HP; ++j) d = fmaf(hi[j], hu[j], d);
    const float z = fmaf(d, sw[ly.out_w], sw[ly.out_b]);
    const float p = sigmoidf_acc(z);
    a.probs[r] = p;
    a.logits[r] = z;
    a.labels[r] = y;
    // backward: dL/dz = (w (p - y)) / B (w = 1 unweighted), the Dot's gradient g = dz w_out, relu' = [a > 0]
    const float dz = row_dz(p, y, a.weight != nullptr, w, a.B);
    if (a.weight) a.weights[r] = w;
#pragma unroll
    for (int q = 0; q < EP / 4; ++q) {
      const float4 mv = ldg4(mrow + 4 * q), uv = ldg4(urow + 4 * q);
      rec[4 * q] = mv.x; rec[4 * q + 1] = mv.y; rec[4 * q + 2] = mv.z; rec[4 * q + 3] = mv.w;
      rec[EP + 4 * q] = uv.x; rec[EP + 4 * q + 1] = uv.y; rec[EP + 4 * q + 2] = uv.z; rec[EP + 4 * q + 3] = uv.w;
    }
    rec[D] = d;
    rec[DZ] = dz;
    const float g = dz * sw[ly.out_w];
#pragma unroll 1
    for (int t = 0; t < 2; ++t) {                       // the item tower, then the user tower
      const float* act = rec + ACT + t * L * HP;
      const float* other = rec + ACT + (1 - t) * L * HP + (L - 1) * HP;   // the other tower's output
      float* dlt = rec + DLT + t * L * HP;
      float dl[HP];
#pragma unroll
      for (int j = 0; j < HP; ++j) dl[j] = act[(L - 1) * HP + j] > 0.f ? g * other[j] : 0.f;
      for (int l = L - 1; l >= 1; --l) {
#pragma unroll
        for (int j = 0; j < HP; ++j) dlt[l * HP + j] = dl[j];
        float dn[HP];
        const float* W = sw + ly.w_off[3 * t + l];
#pragma unroll
        for (int k = 0; k < HP; ++k) {
          float s = 0.f;
#pragma unroll
          for (int j = 0; j < HP; ++j) s = fmaf(W[k * HP + j], dl[j], s);
          dn[k] = act[(l - 1) * HP + k] > 0.f ? s : 0.f;
        }
#pragma unroll
        for (int k = 0; k < HP; ++k) dl[k] = dn[k];
      }
#pragma unroll
      for (int j = 0; j < HP; ++j) dlt[j] = dl[j];
      // the tower's embedding row gradient: W0 . delta_0
      const float* W0 = sw + ly.w_off[3 * t];
      float* ge = a.gemb + (size_t)(t * a.B + r) * EP;
#pragma unroll 4
      for (int k = 0; k < EP; ++k) {
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < HP; ++j) s = fmaf(W0[k * HP + j], dl[j], s);
        ge[k] = s;
      }
    }
    a.trow[r] = mid;
    a.trow[a.B + r] = a.n_movies + uid;
  }
  __syncthreads();
  // Dense gradients of this CTA's rows: parameter q = sum over rows in row order of (input . delta)
  const int nv = min(kTrainRows, a.B - (int)blockIdx.x * kTrainRows);
  for (int q = tid; q < ly.blob_floats; q += kTrainRows) {
    int ao = -2, bo = 0;                               // ao: -2 zero (padding), -1 the constant 1
    for (int t = 0; t < 2; ++t) {
      for (int l = 0; l < L; ++l) {
        const int wo = ly.w_off[3 * t + l], bof = ly.b_off[3 * t + l];
        const int K = l == 0 ? EP : HP;
        if (q >= wo && q < wo + K * HP) {
          const int k = (q - wo) / HP, j = (q - wo) % HP;
          ao = l == 0 ? t * EP + k : ACT + t * L * HP + (l - 1) * HP + k;
          bo = DLT + t * L * HP + l * HP + j;
        } else if (q >= bof && q < bof + HP) {
          ao = -1;
          bo = DLT + t * L * HP + l * HP + (q - bof);
        }
      }
    }
    if (q == ly.out_w) { ao = D; bo = DZ; }
    if (q == ly.out_b) { ao = -1; bo = DZ; }
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
  return (blob_floats + kTrainRows * row_floats(EP, HP, n_layers)) * (int)sizeof(float);
}

template <int EP, int HP>
cudaError_t launch_step_t(const NcfStepArgs* a, const TowerLayout& ly, cudaStream_t s) {
  const int smem = step_smem_bytes(EP, HP, ly.n_layers, ly.blob_floats);
  if (!a)                                             // the opt-in on the current device, no launch
    return cudaFuncSetAttribute(twotowers_train_step_kernel<EP, HP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                smem);
  twotowers_train_step_kernel<EP, HP><<<twotowers_train_ctas(a->B), kTrainRows, smem, s>>>(*a, ly);
  ++g_launch_count;
  return cudaGetLastError();
}

}  // namespace

int twotowers_train_ctas(int B) { return (B + kTrainRows - 1) / kTrainRows; }

cudaError_t launch_twotowers_train_step(const NcfStepArgs* a, const NcfParams& p, cudaStream_t s) {
  TowerLayout ly = tower_layout(p);
  if (!a) {                // the opt-in is at 3 hidden layers, the largest step: each hidden layer past p's adds, per
    ly.blob_floats += 2 * (3 - ly.n_layers) * (p.HP * p.HP + p.HP);   // tower, a kernel [HP][HP] and a bias [HP]
    ly.n_layers = 3;                                                  // (place_ncf)
  }
#define SRS_TT_STEP_CASE(E_, H_) \
  if (p.EP == E_ && p.HP == H_) return launch_step_t<E_, H_>(a, ly, s);
  SRS_TT_STEP_CASE(12, 16) SRS_TT_STEP_CASE(16, 16) SRS_TT_STEP_CASE(32, 16) SRS_TT_STEP_CASE(64, 16)
  SRS_TT_STEP_CASE(12, 32) SRS_TT_STEP_CASE(16, 32) SRS_TT_STEP_CASE(32, 32) SRS_TT_STEP_CASE(64, 32)
#undef SRS_TT_STEP_CASE
  return cudaErrorInvalidValue;
}

}  // namespace srs
