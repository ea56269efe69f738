// metrics.cu - the metrics of Keras's `model.evaluate` over labelled batches (the reference compiles
// every CTR model with loss='binary_crossentropy' and metrics=['accuracy', AUC(curve='ROC'),
// AUC(curve='PR')], e.g. DIN.py:171-181): one kernel folds a batch's scores into a device-resident
// state; the AUCs are computed on the host from that state's 2 x 201 integer counts.
//
// Per row (DESIGN.md section 4, "Metrics"):
//   bin k = #{j : p > t_j} over Keras's 200 float32 thresholds, counted per (label, k);
//   correct = (label == (p > 0.5)), Keras's binary_accuracy;
//   loss = max(x, 0) - x*z + log1p(exp(-|x|)) on the logit x in float32: for a sigmoid output layer
//   Keras's binary_crossentropy takes this logit path, not the clipped-probability formula.
// Counts are integer atomics (exact, order-free).  The loss is reduced in double in a fixed order inside
// each CTA; the last CTA (ticket counter) sums the CTA partials in CTA order, so it has the same bits on
// every run for the same rows.
//
// With sample weights (section 4.28) the same kernel, instantiated with kWeighted, also sums each row's weight into
// its (label, bin), the weighted correct rows and the weights, in double.  No float atomics: a CTA stages each
// 256-row chunk's (bin, weight) pairs in shared memory and thread j adds the weights of bin j in row order; the
// per-CTA sums go to MetricsWeightedReduce and the loss's last CTA adds them in CTA order.  The loss sum becomes
// sum w l through the loss's own reduction, so all-ones weights give the unweighted loss bits.
//
// DIEN's evaluate (DESIGN.md section 4.7) also needs each batch's own histogram (`own_hist`) and, from those,
// auc_value: the mean over batches k of the ROC AUC of batches 0..k (launch_auc_value).
#include <cmath>

#include "../../include/srs_ctr.h"
#include "kernels.h"

namespace srs {

namespace {

constexpr int kMetThreads = 256;
constexpr int kMetRowsPerCta = 4 * kMetThreads;

// Keras's thresholds: [0 - 1e-7] + [(i + 1) / 199 for i in range(198)] + [1 + 1e-7] in double, each cast
// to float32 (IEEE double division and rounding are the same on the device and on the host).
__device__ __forceinline__ float keras_threshold(int j) {
  if (j == 0) return (float)(0.0 - 1e-7);
  if (j == kMetThresholds - 1) return (float)(1.0 + 1e-7);
  return (float)((double)j * 1.0 / (double)(kMetThresholds - 1));
}

constexpr int kMetBinSlots = (2 * kMetBins + kMetThreads - 1) / kMetThreads;   // weighted bins per thread

template <bool kWeighted>
__global__ void __launch_bounds__(kMetThreads)
metrics_update_kernel(const float* __restrict__ probs, const float* __restrict__ logits,
                      const int32_t* __restrict__ labels, int n, MetricsCounters* cnt, MetricsReduce* red,
                      double* loss_dst, int accumulate, unsigned long long* own_hist,
                      const float* __restrict__ weight, MetricsWeighted* wdst, MetricsWeightedReduce* wred) {
  __shared__ float s_t[kMetThresholds];
  __shared__ unsigned int s_hist[2 * kMetBins];
  __shared__ double s_loss[kMetThreads / 32];
  __shared__ unsigned int s_correct;
  __shared__ int s_err;
  __shared__ int s_last;
  __shared__ int s_key[kWeighted ? kMetThreads : 1];          // the chunk's (label, bin) and weight per row
  __shared__ float s_w[kWeighted ? kMetThreads : 1];
  __shared__ double s_wc[kWeighted ? kMetThreads / 32 : 1], s_ws[kWeighted ? kMetThreads / 32 : 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int j = tid; j < kMetThresholds; j += kMetThreads) s_t[j] = keras_threshold(j);
  for (int j = tid; j < 2 * kMetBins; j += kMetThreads) s_hist[j] = 0u;
  if (tid == 0) { s_correct = 0u; s_err = 0; }
  __syncthreads();

  double loss = 0.0;
  unsigned int correct = 0u;
  int err = 0;
  double wbin[kMetBinSlots] = {}, wcorrect = 0.0, wsum = 0.0;   // kWeighted: bins tid + k * kMetThreads
  for (int64_t base = (int64_t)blockIdx.x * kMetThreads; base < n; base += (int64_t)gridDim.x * kMetThreads) {
    const int64_t i = base + tid;
    int key = -1;
    float w = 0.f;
    if (i < n) {
      const float p = __ldg(probs + i);
      const int z = __ldg(labels + i);
      const bool ok_p = p >= 0.f && p <= 1.f;             // false for NaN
      const bool ok_z = z == 0 || z == 1;
      err |= (ok_z ? 0 : kMetErrLabel) | (ok_p ? 0 : kMetErrProb);
      if (ok_p && ok_z) {
        int lo = 0, hi = kMetThresholds;                   // k = #{j : p > t_j}, thresholds ascending
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (p > s_t[mid]) lo = mid + 1; else hi = mid;
        }
        key = z * kMetBins + lo;
        const bool ok = (z == 1) == (p > 0.5f);
        correct += (unsigned int)ok;
        if (kWeighted) {
          w = __ldg(weight + i);
          wsum += (double)w;
          if (ok) wcorrect += (double)w;
          loss += (double)__fmul_rn(w, logit_bce(__ldg(logits + i), z));
        } else {
          loss += (double)logit_bce(__ldg(logits + i), z);
        }
      }
    }
    if (kWeighted) {                                       // bin j's weights in row order, no atomics
      s_key[tid] = key;
      s_w[tid] = w;
      __syncthreads();
      const int rows = (int)min((int64_t)kMetThreads, (int64_t)n - base);
#pragma unroll
      for (int k = 0; k < kMetBinSlots; ++k) {
        const int j = tid + k * kMetThreads;
        for (int r = 0; r < rows; ++r)
          if (s_key[r] == j) wbin[k] += (double)s_w[r];
      }
      __syncthreads();
    }
    // scores cluster: one shared atomic per distinct (label, bin) in the warp
    const unsigned int active = __ballot_sync(0xffffffffu, key >= 0);
    if (key >= 0) {
      const unsigned int peers = __match_any_sync(active, key);
      if (lane == __ffs(peers) - 1) atomicAdd(&s_hist[key], (unsigned int)__popc(peers));
    }
  }

  correct = __reduce_add_sync(0xffffffffu, correct);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
  if (kWeighted) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      wcorrect += __shfl_xor_sync(0xffffffffu, wcorrect, o);
      wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
    }
  }
  err = __reduce_or_sync(0xffffffffu, (unsigned int)err);
  if (lane == 0) {
    s_loss[warp] = loss;
    if (kWeighted) { s_wc[warp] = wcorrect; s_ws[warp] = wsum; }
    if (correct) atomicAdd(&s_correct, correct);
    if (err) atomicOr(&s_err, err);
  }
  __syncthreads();
  if (kWeighted) {                                         // this CTA's weighted sums, before its ticket
    double* part = wred->partial[blockIdx.x];
#pragma unroll
    for (int k = 0; k < kMetBinSlots; ++k)
      if (tid + k * kMetThreads < 2 * kMetBins) part[tid + k * kMetThreads] = wbin[k];
    if (tid == 0) {
      double c = 0.0, s = 0.0;
      for (int w = 0; w < kMetThreads / 32; ++w) { c += s_wc[w]; s += s_ws[w]; }
      part[2 * kMetBins] = c;
      part[2 * kMetBins + 1] = s;
    }
    __threadfence();
    __syncthreads();
  }

  for (int j = tid; j < 2 * kMetBins; j += kMetThreads) {
    const unsigned int v = s_hist[j];
    if (v) atomicAdd(&cnt->hist[j], (unsigned long long)v);
    if (v && own_hist) atomicAdd(&own_hist[j], (unsigned long long)v);
  }
  if (tid == 0) {
    if (s_correct) atomicAdd(&cnt->correct, (unsigned long long)s_correct);
    if (s_err) atomicOr(&cnt->err, s_err);
    double cta = 0.0;
    for (int w = 0; w < kMetThreads / 32; ++w) cta += s_loss[w];
    red->partial[blockIdx.x] = cta;
    __threadfence();
    s_last = atomicAdd(&red->ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (kWeighted) {                                         // the CTAs' weighted sums in CTA order
    double* dst = reinterpret_cast<double*>(wdst);
    for (int q = tid; q < kMetWSums; q += kMetThreads) {
      double t = 0.0;
      for (int b = 0; b < (int)gridDim.x; ++b) t += __ldcg(&wred->partial[b][q]);
      dst[q] = accumulate ? dst[q] + t : t;
    }
  }
  if (warp != 0) return;
  double tot = 0.0;                                        // CTA partials in a fixed order
  for (int b = lane; b < (int)gridDim.x; b += 32) tot += __ldcg(red->partial + b);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
  if (lane == 0) {
    if (loss_dst) *loss_dst = accumulate ? *loss_dst + tot : tot;
    red->ticket = 0u;                                      // ready for the next launch on this stream
  }
}

inline __host__ __device__ double div_no_nan(double a, double b) { return b == 0.0 ? 0.0 : a / b; }

// auc_value of DIEN's evaluate: hist[k] becomes the sum of the batch histograms 0..k (one thread per bin,
// batches in batch order; integer sums, so exact)
__global__ void hist_prefix_kernel(unsigned long long* hist, int K) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= 2 * kMetBins) return;
  unsigned long long c = 0;
  for (int k = 0; k < K; ++k) {
    unsigned long long* h = hist + (size_t)k * 2 * kMetBins + j;
    c += *h;
    *h = c;
  }
}

// auc[k] = the ROC AUC of prefix histogram k, in double: the ROC sum of metrics_summarise, one thread per prefix
__global__ void prefix_auc_kernel(const unsigned long long* __restrict__ hist, int K, double* __restrict__ auc) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const unsigned long long* neg = hist + (size_t)k * 2 * kMetBins;
  const unsigned long long* pos = neg + kMetBins;
  unsigned long long P = 0, N = 0;
  for (int j = 0; j < kMetBins; ++j) { P += pos[j]; N += neg[j]; }
  unsigned long long above_p = P - pos[0], above_n = N - neg[0];
  double r0 = div_no_nan((double)above_p, (double)P), f0 = div_no_nan((double)above_n, (double)N);
  double roc = 0.0;
  for (int j = 1; j < kMetThresholds; ++j) {
    above_p -= pos[j]; above_n -= neg[j];
    const double r1 = div_no_nan((double)above_p, (double)P), f1 = div_no_nan((double)above_n, (double)N);
    roc += (f0 - f1) * ((r0 + r1) / 2.0);
    r0 = r1; f0 = f1;
  }
  auc[k] = roc;
}

// *dst = sum of v[0..K) in a fixed order (one warp: strided lane sums, then a fixed butterfly)
__global__ void ordered_sum_kernel(const double* __restrict__ v, int K, double* dst) {
  double s = 0.0;
  for (int k = threadIdx.x; k < K; k += 32) s += v[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (threadIdx.x == 0) *dst = s;
}

}  // namespace

cudaError_t launch_metrics_update(const float* probs, const float* logits, const int32_t* labels, int n,
                                  MetricsCounters* cnt, MetricsReduce* red, double* loss_dst, int accumulate,
                                  cudaStream_t s, unsigned long long* own_hist) {
  if (n <= 0) return cudaSuccess;
  int64_t blocks = ((int64_t)n + kMetRowsPerCta - 1) / kMetRowsPerCta;
  if (blocks > kMetMaxCtas) blocks = kMetMaxCtas;
  metrics_update_kernel<false><<<(int)blocks, kMetThreads, 0, s>>>(probs, logits, labels, n, cnt, red, loss_dst,
                                                                   accumulate, own_hist, nullptr, nullptr, nullptr);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_metrics_update_weighted(const float* probs, const float* logits, const int32_t* labels,
                                           const float* w, int n, MetricsCounters* cnt, MetricsReduce* red,
                                           double* loss_dst, MetricsWeighted* wdst, MetricsWeightedReduce* wred,
                                           int accumulate, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  int64_t blocks = ((int64_t)n + kMetRowsPerCta - 1) / kMetRowsPerCta;
  if (blocks > kMetMaxCtas) blocks = kMetMaxCtas;
  metrics_update_kernel<true><<<(int)blocks, kMetThreads, 0, s>>>(probs, logits, labels, n, cnt, red, loss_dst,
                                                                  accumulate, nullptr, w, wdst, wred);
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_auc_value(unsigned long long* hist, int K, double* auc, double* sum_dst, cudaStream_t s) {
  if (K <= 0) return cudaSuccess;
  hist_prefix_kernel<<<(2 * kMetBins + 127) / 128, 128, 0, s>>>(hist, K);
  prefix_auc_kernel<<<(K + 127) / 128, 128, 0, s>>>(hist, K, auc);
  ordered_sum_kernel<<<1, 32, 0, s>>>(auc, K, sum_dst);
  g_launch_count += 3;
  return cudaGetLastError();
}

// Keras's AUC(num_thresholds=200, summation_method='interpolation') of the TP/FP/TN/FN per threshold, into
// out->roc_auc and out->pr_auc
static void auc_sums(const double* tp, const double* fp, const double* tn, const double* fn, srs_eval_result* out) {
  double roc = 0.0, pr = 0.0;
  for (int j = 0; j + 1 < kMetThresholds; ++j) {
    const double r0 = div_no_nan(tp[j], tp[j] + fn[j]), r1 = div_no_nan(tp[j + 1], tp[j + 1] + fn[j + 1]);
    const double f0 = div_no_nan(fp[j], fp[j] + tn[j]), f1 = div_no_nan(fp[j + 1], fp[j + 1] + tn[j + 1]);
    roc += (f0 - f1) * ((r0 + r1) / 2.0);
    // interpolate_pr_auc (Davis & Goadrich 2006)
    const double dtp = tp[j] - tp[j + 1];
    const double p0 = tp[j] + fp[j], p1 = tp[j + 1] + fp[j + 1];
    const double dp = p0 - p1;
    const double slope = div_no_nan(dtp, std::fmax(dp, 0.0));
    const double intercept = tp[j + 1] - slope * p1;
    const double ratio = (p0 > 0.0 && p1 > 0.0) ? div_no_nan(p0, std::fmax(p1, 0.0)) : 1.0;
    pr += div_no_nan(slope * (dtp + intercept * std::log(ratio)), std::fmax(tp[j + 1] + fn[j + 1], 0.0));
  }
  out->roc_auc = roc;
  out->pr_auc = pr;
}

// Keras's AUC(num_thresholds=200, summation_method='interpolation') from the (label, bin) counts.  Keras
// keeps TP/FP/TN/FN in float32 variables, which stop being exact above 2^24 rows; these are exact integers.
void metrics_summarise(const unsigned long long* hist, unsigned long long correct, double loss_sum,
                       srs_eval_result* out, int64_t* confusion) {
  const unsigned long long* neg = hist;
  const unsigned long long* pos = hist + kMetBins;
  double tp[kMetThresholds], fp[kMetThresholds], tn[kMetThresholds], fn[kMetThresholds];
  unsigned long long P = 0, N = 0;
  for (int k = 0; k < kMetBins; ++k) { P += pos[k]; N += neg[k]; }
  unsigned long long above_p = P, above_n = N;             // rows with bin > j, i.e. p > t_j
  for (int j = 0; j < kMetThresholds; ++j) {
    above_p -= pos[j]; above_n -= neg[j];
    tp[j] = (double)above_p; fp[j] = (double)above_n;
    fn[j] = (double)(P - above_p); tn[j] = (double)(N - above_n);
    if (confusion) {
      confusion[j] = (int64_t)above_p;
      confusion[kMetThresholds + j] = (int64_t)above_n;
      confusion[2 * kMetThresholds + j] = (int64_t)(N - above_n);
      confusion[3 * kMetThresholds + j] = (int64_t)(P - above_p);
    }
  }
  const unsigned long long rows = P + N;
  out->rows = (int64_t)rows;
  out->positives = (int64_t)P;
  out->correct = (int64_t)correct;
  out->loss = rows ? loss_sum / (double)rows : 0.0;
  out->accuracy = rows ? (double)correct / (double)rows : 0.0;
  auc_sums(tp, fp, tn, fn, out);
}

void metrics_summarise_weighted(const unsigned long long* hist, unsigned long long correct, const MetricsWeighted& w,
                                double loss_sum, srs_eval_result* out) {
  metrics_summarise(hist, correct, loss_sum, out, nullptr);     // rows, positives, correct and the loss
  const double* neg = w.hist;
  const double* pos = w.hist + kMetBins;
  // tp[j] / fp[j]: the weights of the rows with bin > j, summed from the top bin down; fn / tn from bin 0 up.
  // Integer weights give exact sums, so all-ones weights give the counts' bits.
  double tp[kMetThresholds], fp[kMetThresholds], tn[kMetThresholds], fn[kMetThresholds];
  double above_p = 0.0, above_n = 0.0, below_p = 0.0, below_n = 0.0;
  for (int j = kMetThresholds - 1; j >= 0; --j) {
    above_p += pos[j + 1]; above_n += neg[j + 1];
    tp[j] = above_p; fp[j] = above_n;
  }
  for (int j = 0; j < kMetThresholds; ++j) {
    below_p += pos[j]; below_n += neg[j];
    fn[j] = below_p; tn[j] = below_n;
  }
  out->accuracy = div_no_nan(w.correct, w.sum);
  auc_sums(tp, fp, tn, fn, out);
}

}  // namespace srs
