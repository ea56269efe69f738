// deepfm2_train.cu - the forward / backward step of DeepFM_v2's `model.fit` (DeepFM_v2.py:158-165); the trainer
// that drives it (permutation, dedupe, Adam, metrics) is srs_trainer in trainer.cu.  DESIGN.md section 4.19.
//
// deepfm2_train_step_kernel<EP>: one 32-row tile per CTA, 256 threads.  The forward is deepfm2_kernel's
// (deepfm2_layers.cuh), so a step's outputs are the serving outputs bit for bit.  The backward runs on the same
// tile:
//   dz      = (sigmoid(z) - y) / B per row;  dfirst = dz * out/kernel[0]
//   delta2  = dz * out/kernel[65 + j] where a2 > 0;  delta1 = Wd1 . delta2 where a1 > 0
//   dF      = Wd . delta1 + dz * out/kernel[1 + c] * 2 (s_c - F_fc), s_c = sum_f F_fc
//   entries each row's 4 table rows (a missing genre writes none) with their gradients proj_f . dF_f, and its 4
//           one-hot rows of first_cat/kernel (scalar dfirst), for table_grad_kernel to dedupe in row order
//   partial thread q sums Dense parameter q's gradient over the CTA's rows in row order
// No float atomics.  The trainer's forward for validation and evaluate is deepfm2_kernel itself (launch_deepfm2).
#include "deepfm2_layers.cuh"

namespace srs {

namespace {

constexpr int kFm2StepRows = 32;   // rows per CTA of the step: a 64-row tile and its backward do not fit at EP = 64
constexpr int kLDM = kProj + 4;    // the FM terms' tile [R][kLDM]

// the forward tile | dF [R][LDF] | delta1 [R][LD1] | delta2 [R][LD2] | FM terms [R][kLDM] | first, dfirst, dz [R]
template <int EP>
constexpr int step_smem_floats() {
  using T = DeepFm2Tile<EP, kFm2StepRows>;
  return T::kFloats + kFm2StepRows * (T::LDF + T::LD1 + T::LD2 + kLDM + 3);
}
static_assert(step_smem_floats<64>() * 4 <= 227 * 1024, "the EP = 64 step tile must fit in shared memory");

template <int EP>
__global__ void __launch_bounds__(kThreads) deepfm2_train_step_kernel(DeepFm2StepArgs a) {
  using T = DeepFm2Tile<EP, kFm2StepRows>;
  constexpr int R = T::R, LDX = T::LDX, LDF = T::LDF, LD1 = T::LD1, LD2 = T::LD2;
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem + T::kXs;
  float* Fs = smem + T::kFs;
  float* H1 = smem + T::kH1;
  float* H2 = smem + T::kH2;
  float* Wds = smem + T::kWds;
  float* Wd1s = smem + T::kWd1s;
  float* dF = smem + T::kFloats;                 // dL/dF
  float* D1 = dF + R * LDF;                      // delta of the first hidden layer
  float* D2 = D1 + R * LD1;                      // delta of the second
  float* FMs = D2 + R * LD2;                     // the FM terms
  float* firsts = FMs + R * kLDM;                // the first-order value
  float* dfs = firsts + R;                       // dL/dfirst
  float* dzs = dfs + R;                          // dL/dz
  const DeepFm2Blob ly = DeepFm2Blob::of(EP);
  const BatchView& b = a.io.b;
  const DeepFm2Params& p = a.p;
  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * R;
  const int nv = min(R, b.B - row0);

  stage_weights(Wds, p.Wd, 5 * kProj * 32);
  stage_weights(Wd1s, p.Wd1, 32 * 16);
  deepfm2_tile_gather<EP, R>(p, b, row0, Xs);
  __syncthreads();
  deepfm2_tile_project<EP, R>(p, Xs, Fs);
  __syncthreads();
  stage_wait();
  __syncthreads();
  deepfm2_tile_mlp<EP, R>(p, Fs, Wds, Wd1s, H1, H2);
  deepfm2_tile_logits<EP, R, true>(p, b, row0, Xs, Fs, H2, FMs, kLDM, firsts, [&](int r, int row, float z) {
    const float pr = sigmoidf_acc(z);
    b.probs[row] = pr;
    b.logits[row] = z;
    const float dz = row_dz(pr, __ldg(a.io.label + row), a.io.weight, row, b.B);
    dzs[r] = dz;
    dfs[r] = dz * __ldg(p.wout);
  });
  __syncthreads();
  for (int i = tid; i < nv * 16; i += kThreads) {
    const int r = i >> 4, j = i & 15;
    D2[r * LD2 + j] = H2[r * LD2 + j] > 0.f ? dzs[r] * __ldg(p.wout + 1 + kProj + j) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < nv * 32; i += kThreads) {
    const int r = i >> 5, k = i & 31;
    float s = 0.f;
    for (int j = 0; j < 16; ++j) s = fmaf(Wd1s[k * 16 + j], D2[r * LD2 + j], s);
    D1[r * LD1 + k] = H1[r * LD1 + k] > 0.f ? s : 0.f;
  }
  __syncthreads();
  // dF: the deep part Wd . delta1, then the FM part
  for (int i = tid; i < nv * 5 * kProj; i += kThreads) {
    const int r = i / (5 * kProj), q = i % (5 * kProj), c = q & (kProj - 1);
    const float* f = Fs + r * LDF;
    float s = 0.f;
    for (int kk = 0; kk < 32; ++kk) {            // k rotated by q: the lanes of a warp hit distinct banks
      const int k = (kk + q) & 31;
      s = fmaf(Wds[q * 32 + k], D1[r * LD1 + k], s);
    }
    float sc = 0.f;
#pragma unroll
    for (int g = 0; g < 5; ++g) sc += f[g * kProj + c];
    dF[r * LDF + q] = s + dzs[r] * __ldg(p.wout + 1 + c) * 2.f * (sc - f[q]);
  }
  __syncthreads();

  // table and one-hot entries: field s of tile row r is entry s * B + row
  for (int i = tid; i < nv * kDeepFm2Tables; i += kThreads) {
    const int r = i / kDeepFm2Tables, s = i % kDeepFm2Tables;
    const int row = row0 + r;
    const int G = p.n_genres;
    int id, off;                                 // off: the field's first row in first_cat/kernel
    switch (s) {
      case 0: id = __ldg(b.movie_genre + row * 3); off = 0; break;
      case 1: id = __ldg(b.movie_id + row); off = G; break;
      case 2: id = __ldg(b.user_genre + row * 5); off = G + p.n_movies; break;
      default: id = __ldg(b.user_id + row); off = 2 * G + p.n_movies; break;
    }
    a.io.trow[s * b.B + row] = id < 0 ? -1 : (int32_t)(a.tab_row0[s] + id);
    a.io.frow[s * b.B + row] = id < 0 ? -1 : off + id;
    a.io.fgrad[s * b.B + row] = dfs[r];
  }
  // their gradients: row k of proj_f against each row's dF_f, one warp per (f, k), the proj row read once
  const int warp = tid >> 5, lane = tid & 31;
  for (int q = warp; q < kDeepFm2Tables * EP; q += kThreads / 32) {
    const int f = q / EP, k = q % EP;
    const float2 w = __ldg(reinterpret_cast<const float2*>(p.blob + ly.proj + (size_t)q * kProj) + lane);
    for (int r = 0; r < nv; ++r) {
      const float2 d = *reinterpret_cast<const float2*>(dF + r * LDF + f * kProj + 2 * lane);
      float g = fmaf(w.y, d.y, w.x * d.x);
      g = warp_sum(g);
      if (lane == 0) a.io.gemb[((size_t)f * b.B + row0 + r) * EP + k] = g;
    }
  }

  // Dense gradients of this CTA's rows: parameter q = sum over rows in row order of (input . delta)
  for (int q = tid; q < ly.floats; q += kThreads) {
    const float* in = nullptr;                   // null: the constant 1 (a bias)
    const float* dl = nullptr;                   // null: no gradient (padding)
    int ldi = 0, ldd = 0;
    if (q < ly.proj_b) {                         // proj_f/kernel [f][k][c]
      const int f = q / (EP * kProj), k = (q / kProj) % EP, c = q % kProj;
      in = Xs + f * EP + k; ldi = LDX; dl = dF + f * kProj + c; ldd = LDF;
    } else if (q < ly.proj_num) {
      dl = dF + (q - ly.proj_b); ldd = LDF;
    } else if (q < ly.proj_num_b) {
      in = Xs + 4 * EP + (q - ly.proj_num) / kProj; ldi = LDX; dl = dF + 4 * kProj + (q - ly.proj_num) % kProj; ldd = LDF;
    } else if (q < ly.Wd) {
      dl = dF + 4 * kProj + (q - ly.proj_num_b); ldd = LDF;
    } else if (q < ly.bd) {
      in = Fs + (q - ly.Wd) / 32; ldi = LDF; dl = D1 + (q - ly.Wd) % 32; ldd = LD1;
    } else if (q < ly.Wd1) {
      dl = D1 + (q - ly.bd); ldd = LD1;
    } else if (q < ly.bd1) {
      in = H1 + (q - ly.Wd1) / 16; ldi = LD1; dl = D2 + (q - ly.Wd1) % 16; ldd = LD2;
    } else if (q < ly.wout) {
      dl = D2 + (q - ly.bd1); ldd = LD2;
    } else if (q < ly.first_num) {               // out/kernel: first | fm | deep, then padding
      const int j = q - ly.wout;
      if (j < 1 + kProj + 16) { dl = dzs; ldd = 1; }
      if (j == 0) { in = firsts; ldi = 1; }
      else if (j < 1 + kProj) { in = FMs + (j - 1); ldi = kLDM; }
      else { in = H2 + (j - 1 - kProj); ldi = LD2; }
    } else if (q < ly.first_cat_b) {             // first_num/kernel
      in = Xs + 4 * EP + (q - ly.first_num); ldi = LDX; dl = dfs; ldd = 1;
    } else if (q < ly.bout) {                    // first_cat/bias, first_num/bias
      dl = dfs; ldd = 1;
    } else if (q == ly.bout) {
      dl = dzs; ldd = 1;
    }
    float s = 0.f;
    if (dl && in) {
      for (int r = 0; r < nv; ++r) s = fmaf(in[r * ldi], dl[r * ldd], s);
    } else if (dl) {
      for (int r = 0; r < nv; ++r) s += dl[r * ldd];
    }
    a.io.part[(size_t)blockIdx.x * ly.floats + q] = s;
  }
}

template <int EP>
cudaError_t launch_step_t(const DeepFm2StepArgs* a, cudaStream_t s) {
  constexpr int smem = step_smem_floats<EP>() * (int)sizeof(float);
  if (!a)                                             // the opt-in on the current device, no launch
    return cudaFuncSetAttribute(deepfm2_train_step_kernel<EP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  deepfm2_train_step_kernel<EP><<<deepfm2_train_ctas(a->io.b.B), kThreads, smem, s>>>(*a);
  ++g_launch_count;
  return cudaGetLastError();
}

}  // namespace

int deepfm2_train_ctas(int B) { return (B + kFm2StepRows - 1) / kFm2StepRows; }

cudaError_t launch_deepfm2_train_step(int EP, const DeepFm2StepArgs* a, cudaStream_t s) {
#define SRS_FM2_STEP_CASE(E_) \
  if (EP == E_) return launch_step_t<E_>(a, s);
  SRS_FM2_STEP_CASE(12) SRS_FM2_STEP_CASE(16) SRS_FM2_STEP_CASE(32) SRS_FM2_STEP_CASE(64)
#undef SRS_FM2_STEP_CASE
  return cudaErrorInvalidValue;
}

}  // namespace srs
