// ncf.cu - NeuralCF (neural_cf_model_1) and two-tower (neural_cf_model_2) forward.
//
// Reference: TFRecModel/src/com/sparrowrecsys/offline/tensorflow/NeuralCF.py:45-70.
// 92 algorithmic bytes and ~600 FLOP per row: the path is two scattered row gathers
// and a score store, so the kernel is one thread per row (each thread issues its
// 2*EP/4 independent 128-bit loads up front), Dense weights broadcast from shared
// memory, nothing staged per row.
#include "kernels.h"
#include "ncf_layers.cuh"

namespace srs {

template <int EP, int HP>
__global__ void __launch_bounds__(128) ncf_kernel(NcfParams p, BatchView b) {
  extern __shared__ __align__(16) float sw[];
  for (int i = threadIdx.x; i < p.blob_floats; i += blockDim.x) sw[i] = __ldg(p.blob + i);
  __syncthreads();
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= b.B) return;
  const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
  const int uid = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
  const float* mrow = p.movie + (size_t)mid * EP;
  const float* urow = p.user + (size_t)uid * EP;

  float z;
  if (!p.two_towers) {
    float h[HP];
#pragma unroll
    for (int j = 0; j < HP; ++j) h[j] = sw[p.b_off[0] + j];
    first_layer_accum<EP, HP>(h, mrow, sw + p.w_off[0]);                // item rows first
    first_layer_accum<EP, HP>(h, urow, sw + p.w_off[0] + EP * HP);      // then user rows
#pragma unroll
    for (int j = 0; j < HP; ++j) h[j] = fmaxf(h[j], 0.f);
    for (int l = 1; l < p.n_layers; ++l) hidden_layer<HP>(h, sw + p.w_off[l], sw + p.b_off[l]);
    z = sw[p.out_b];
#pragma unroll
    for (int j = 0; j < HP; ++j) z = fmaf(h[j], sw[p.out_w + j], z);
    store_score(b, row, sigmoidf_acc(z));
    if (b.logits) b.logits[row] = z;
  } else {
    float hi[HP], hu[HP];
#pragma unroll
    for (int j = 0; j < HP; ++j) { hi[j] = sw[p.b_off[0] + j]; hu[j] = sw[p.b_off[3] + j]; }
    first_layer_accum<EP, HP>(hi, mrow, sw + p.w_off[0]);
    first_layer_accum<EP, HP>(hu, urow, sw + p.w_off[3]);
#pragma unroll
    for (int j = 0; j < HP; ++j) { hi[j] = fmaxf(hi[j], 0.f); hu[j] = fmaxf(hu[j], 0.f); }
    for (int l = 1; l < p.n_layers; ++l) {
      hidden_layer<HP>(hi, sw + p.w_off[l], sw + p.b_off[l]);
      hidden_layer<HP>(hu, sw + p.w_off[3 + l], sw + p.b_off[3 + l]);
    }
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < HP; ++j) d = fmaf(hi[j], hu[j], d);
    if (p.final_dense) {
      z = fmaf(d, sw[p.out_w], sw[p.out_b]);
      store_score(b, row, sigmoidf_acc(z));
    } else {
      z = d;                                   // shipped MLPRec/005: raw Dot output
      store_score(b, row, d);
    }
    if (b.logits) b.logits[row] = z;
  }
}

template <int EP, int HP>
static cudaError_t launch_ncf_t(const NcfParams& p, const BatchView& b, cudaStream_t s) {
  const int threads = 128;
  const int blocks = (b.B + threads - 1) / threads;
  const size_t smem = (size_t)p.blob_floats * sizeof(float);
  ncf_kernel<EP, HP><<<blocks, threads, smem, s>>>(p, b);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_ncf(const NcfParams& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
#define SRS_NCF_CASE(E_, H_) \
  if (p.EP == E_ && p.HP == H_) return launch_ncf_t<E_, H_>(p, b, s);
  SRS_NCF_CASE(12, 16) SRS_NCF_CASE(16, 16) SRS_NCF_CASE(32, 16) SRS_NCF_CASE(64, 16)
  SRS_NCF_CASE(12, 32) SRS_NCF_CASE(16, 32) SRS_NCF_CASE(32, 32) SRS_NCF_CASE(64, 32)
#undef SRS_NCF_CASE
  return cudaErrorInvalidValue;
}

}  // namespace srs
