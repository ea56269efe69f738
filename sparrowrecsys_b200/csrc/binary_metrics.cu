// binary_metrics.cu - mllib's BinaryClassificationMetrics (Spark 2.4.3; OFF/evaluate/Evaluator.scala) over many
// score sets in one call.  DESIGN.md section 4.22 gives the semantics; oracle/binary_metrics.py restates them.
//
//   keys    bm_keys_kernel: each score's descending key in Double.compare's order (NaN first, 0.0 above -0.0)
//           and a tag (set << 1 | positive);
//   sort    a CUB radix sort of (key, tag) (key bits 29..63 for float32 scores), then - with more than one set -
//           a stable radix sort on the tag's set bits: the pairs in (set, descending score) order;
//   runs    bm_heads_kernel flags each run's first pair and writes the positive bits, DeviceSelect keeps the run
//           starts and an inclusive scan turns the bits into cumulative positive counts (exact integers);
//   points  bm_sets_kernel finds each set's first run and positive count; the host bins each set's runs
//           (grouping = runs / numBins) and lays out the points; bm_points_kernel writes each point's threshold
//           and cumulative TP / FP;
//   areas   bm_area_chunk_kernel sums the ROC and PR trapezoids of kChunk consecutive points of one set, each
//           thread's slice in order and then a block reduction; bm_area_set_kernel adds a set's chunks in a
//           fixed order and ROC's last segment to (1, 1).
// The curves are written on request from the points kept on the device (bm_curve_kernel).  No float atomics: the
// same inputs give the same bits.  Every entry point checks its arguments before any device call.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <cstring>
#include <memory>
#include <new>
#include <vector>

#include "../../include/srs_ctr.h"
#include "double_key.cuh"
#include "hostcall.h"

struct srs_binary_metrics {
  int32_t device = 0;
  int32_t n_sets = 0;
  std::vector<int64_t> n, positives, pt_off;     // per set; pt_off [n_sets + 1]
  std::vector<double> roc, pr;
  double* thr = nullptr;                         // device, [pt_off[n_sets]] each
  int64_t* tp = nullptr;
  int64_t* fp = nullptr;
  ~srs_binary_metrics() {
    if (thr || tp || fp) cudaSetDevice(device);
    cudaFree(thr);
    cudaFree(tp);
    cudaFree(fp);
  }
};

namespace srs {
namespace {

constexpr int64_t kMaxPairs = 2147483647;        // int32 positions; the tag holds set << 1 below 2^32
constexpr int kChunk = 2048;                     // points per block of bm_area_chunk_kernel
constexpr int kChunkThreads = 256;
constexpr int kPerThread = kChunk / kChunkThreads;

#define BM_GRID_STRIDE(i, n) \
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// Spark's threshold order is desc_key's (double_key.cuh): Double.compare descending, every NaN one key (0, first)

// BinaryLabelCounter: a label > 0.5 is a positive (a NaN label is not)
__device__ __forceinline__ uint32_t positive(double y) { return y > 0.5 ? 1u : 0u; }
__device__ __forceinline__ uint32_t positive(int32_t y) { return y > 0 ? 1u : 0u; }

// the metric computers: IEEE divisions of exact counts
__host__ __device__ __forceinline__ double precision_of(int64_t tp, int64_t fp) {
  return tp + fp == 0 ? 1.0 : (double)tp / (double)(tp + fp);
}
__host__ __device__ __forceinline__ double rate_of(int64_t c, int64_t total) {
  return total == 0 ? 0.0 : (double)c / (double)total;
}
__device__ __forceinline__ double f_measure_of(double p, double r, double beta) {   // no contraction into an FMA
  const double b2 = __dmul_rn(beta, beta);
  return p + r == 0 ? 0.0 : __dmul_rn(1.0 + b2, __dmul_rn(p, r) / __dadd_rn(__dmul_rn(b2, p), r));
}
// AreaUnderCurve.trapezoid
__host__ __device__ __forceinline__ double trapezoid(double x1, double y1, double x2, double y2) {
  return (x2 - x1) * (y2 + y1) / 2.0;
}

// the last index i of off[0 .. m] with off[i] <= v (off ascending, off[0] <= v)
template <class T>
__device__ __forceinline__ int upper_index(const T* off, int m, int64_t v) {
  int lo = 0, hi = m;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if ((int64_t)off[mid] <= v) lo = mid; else hi = mid;
  }
  return lo;
}

template <class S, class L>
__global__ void bm_keys_kernel(const S* __restrict__ score, const L* __restrict__ label, int n,
                               const int64_t* __restrict__ set_off, int n_sets, uint64_t* __restrict__ key,
                               uint32_t* __restrict__ tag) {
  BM_GRID_STRIDE(i, n) {
    const uint32_t s = n_sets == 1 ? 0u : (uint32_t)upper_index(set_off, n_sets, i);
    key[i] = desc_key((double)score[i]);
    tag[i] = (s << 1) | positive(label[i]);
  }
}

// head[i]: pair i starts a run of equal (set, key); pos[i]: its positive bit (scanned in place afterwards)
__global__ void bm_heads_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ tag, int n,
                                uint8_t* __restrict__ head, int32_t* __restrict__ pos) {
  BM_GRID_STRIDE(i, n) {
    const uint32_t t = tag[i];
    head[i] = i == 0 || key[i] != key[i - 1] || (t >> 1) != (tag[i - 1] >> 1);
    pos[i] = (int32_t)(t & 1u);
  }
}

// per set: its first run (run_off [n_sets + 1]) and its positives, from the cumulative positive counts `cum`
__global__ void bm_sets_kernel(const int64_t* __restrict__ set_off, int n_sets, const int32_t* __restrict__ run_start,
                               const int* __restrict__ n_runs, const int32_t* __restrict__ cum,
                               int64_t* __restrict__ run_off, int64_t* __restrict__ positives) {
  BM_GRID_STRIDE(s, n_sets) {
    const int64_t b = set_off[s], e = set_off[s + 1];
    int lo = 0, hi = *n_runs;                    // the run starting at b
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (run_start[mid] < b) lo = mid + 1; else hi = mid;
    }
    run_off[s] = lo;
    positives[s] = (int64_t)cum[e - 1] - (b ? cum[b - 1] : 0);
    if (s == 0) run_off[n_sets] = *n_runs;
  }
}

struct PointArgs {
  const int64_t* pt_off;                         // [n_sets + 1]
  const int32_t* grouping;                       // [n_sets]
  const int64_t* run_off;                        // [n_sets + 1]
  const int64_t* set_off;                        // [n_sets + 1]
  int n_sets;
};

// point p of set s, local j: runs [run_off[s] + j g, min(run_off[s] + (j + 1) g, run_off[s + 1])) merged; the
// threshold is the first run's score, the counts cumulative to the last run's end
__global__ void bm_points_kernel(PointArgs a, int64_t n_points, const int32_t* __restrict__ run_start,
                                 const uint64_t* __restrict__ key, const int32_t* __restrict__ cum,
                                 double* __restrict__ thr, int64_t* __restrict__ tp, int64_t* __restrict__ fp) {
  BM_GRID_STRIDE(p, n_points) {
    const int s = upper_index(a.pt_off, a.n_sets, p);
    const int64_t g = a.grouping[s];
    const int64_t r0 = a.run_off[s] + (p - a.pt_off[s]) * g;
    const int64_t r1 = min(r0 + g, a.run_off[s + 1]);
    const int64_t start = a.set_off[s];
    const int64_t end = (r1 == a.run_off[s + 1] ? a.set_off[s + 1] : (int64_t)run_start[r1]) - 1;
    const int64_t t = (int64_t)cum[end] - (start ? cum[start - 1] : 0);
    thr[p] = key_score(key[run_start[r0]]);
    tp[p] = t;
    fp[p] = end - start + 1 - t;
  }
}

struct AreaArgs {
  const int64_t* pt_off;                         // [n_sets + 1]
  const int64_t* ch_off;                         // [n_sets + 1]: set s's chunks
  const int64_t* positives;                      // [n_sets]
  const int64_t* set_off;                        // [n_sets + 1]
  int n_sets;
};

// one block per chunk of kChunk points of one set: thread t adds the trapezoids of points t * kPerThread ..
// (t + 1) * kPerThread - 1 in order, then the block's fixed reduction -> part_roc / part_pr [chunk]
__global__ void __launch_bounds__(kChunkThreads) bm_area_chunk_kernel(AreaArgs a, const int64_t* __restrict__ tp,
                                                                        const int64_t* __restrict__ fp,
                                                                        double* __restrict__ part_roc,
                                                                        double* __restrict__ part_pr) {
  const int64_t c = blockIdx.x;
  const int s = upper_index(a.ch_off, a.n_sets, c);
  const int64_t first = a.pt_off[s], last = a.pt_off[s + 1];
  const int64_t P = a.positives[s], N = a.set_off[s + 1] - a.set_off[s] - P;
  const int64_t b = first + (c - a.ch_off[s]) * kChunk + (int64_t)threadIdx.x * kPerThread;
  double roc = 0.0, pr = 0.0;
  for (int64_t p = b; p < b + kPerThread && p < last; ++p) {
    const double prec = precision_of(tp[p], fp[p]), rec = rate_of(tp[p], P), fpr = rate_of(fp[p], N);
    double prec0 = prec, rec0 = 0.0, fpr0 = 0.0;   // the curves' first points: (0, prec) and (0, 0)
    if (p > first) {
      prec0 = precision_of(tp[p - 1], fp[p - 1]);
      rec0 = rate_of(tp[p - 1], P);
      fpr0 = rate_of(fp[p - 1], N);
    }
    roc += trapezoid(fpr0, rec0, fpr, rec);
    pr += trapezoid(rec0, prec0, rec, prec);
  }
  using BR = cub::BlockReduce<double, kChunkThreads>;
  __shared__ typename BR::TempStorage t1, t2;
  const double sr = BR(t1).Sum(roc), sp = BR(t2).Sum(pr);
  if (threadIdx.x == 0) {
    part_roc[c] = sr;
    part_pr[c] = sp;
  }
}

// one warp per set: lane l adds chunks l, l + 32, ... in order, then a fixed shuffle tree, then ROC's segment from
// the last point to (1, 1)
__global__ void bm_area_set_kernel(AreaArgs a, const int64_t* __restrict__ tp, const int64_t* __restrict__ fp,
                                   const double* __restrict__ part_roc, const double* __restrict__ part_pr,
                                   double* __restrict__ roc, double* __restrict__ pr) {
  const int lane = threadIdx.x & 31;
  const int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (s >= a.n_sets) return;
  double r = 0.0, q = 0.0;
  for (int64_t c = a.ch_off[s] + lane; c < a.ch_off[s + 1]; c += 32) {
    r += part_roc[c];
    q += part_pr[c];
  }
  for (int o = 16; o > 0; o >>= 1) {
    r += __shfl_down_sync(0xffffffffu, r, o);
    q += __shfl_down_sync(0xffffffffu, q, o);
  }
  if (lane == 0) {
    const int64_t last = a.pt_off[s + 1] - 1;
    const int64_t P = a.positives[s], N = a.set_off[s + 1] - a.set_off[s] - P;
    roc[s] = r + trapezoid(rate_of(fp[last], N), rate_of(tp[last], P), 1.0, 1.0);
    pr[s] = q;
  }
}

// curve `which` of the set whose points are [first, first + T): out as the header lays it out
__global__ void bm_curve_kernel(int which, double beta, int64_t first, int64_t T, int64_t P, int64_t N,
                                const double* __restrict__ thr, const int64_t* __restrict__ tp,
                                const int64_t* __restrict__ fp, double* __restrict__ out) {
  const int64_t len = which == SRS_BM_ROC ? T + 2 : which == SRS_BM_PR ? T + 1 : T;
  BM_GRID_STRIDE(q, len) {
    if (which == SRS_BM_ROC) {
      if (q == 0 || q == T + 1) {
        out[2 * q] = out[2 * q + 1] = q == 0 ? 0.0 : 1.0;
      } else {
        const int64_t p = first + q - 1;
        out[2 * q] = rate_of(fp[p], N);
        out[2 * q + 1] = rate_of(tp[p], P);
      }
    } else if (which == SRS_BM_PR) {
      const int64_t p = first + (q == 0 ? 0 : q - 1);
      out[2 * q] = q == 0 ? 0.0 : rate_of(tp[p], P);
      out[2 * q + 1] = precision_of(tp[p], fp[p]);
    } else if (which == SRS_BM_THRESHOLDS) {
      out[q] = thr[first + q];
    } else {
      const int64_t p = first + q;
      const double prec = precision_of(tp[p], fp[p]), rec = rate_of(tp[p], P);
      out[2 * q] = thr[p];
      out[2 * q + 1] = which == SRS_BM_PRECISION ? prec : which == SRS_BM_RECALL ? rec
                                                                                 : f_measure_of(prec, rec, beta);
    }
  }
}

int check_args(const void* scores, const void* labels, int64_t n, const int64_t* set_off, int32_t n_sets,
               int32_t num_bins, srs_binary_metrics** out) {
  if (!out) return failf(SRS_ERR_INVALID, "binary metrics: null output handle");
  if (!scores || !labels) return failf(SRS_ERR_INVALID, "binary metrics: null scores or labels");
  if (n < 1 || n > kMaxPairs)
    return failf(SRS_ERR_INVALID, "binary metrics: n = %lld pairs, must be 1 .. %lld", (long long)n,
                 (long long)kMaxPairs);
  if (num_bins < 0) return failf(SRS_ERR_INVALID, "binary metrics: num_bins = %d must be >= 0", num_bins);
  if (set_off) {
    if (n_sets < 1 || n_sets > n)
      return failf(SRS_ERR_INVALID, "binary metrics: n_sets = %d, must be 1 .. n", n_sets);
    if (set_off[0] != 0 || set_off[n_sets] != n)
      return failf(SRS_ERR_INVALID, "binary metrics: set offsets must run from 0 to n = %lld", (long long)n);
    for (int32_t s = 0; s < n_sets; ++s)
      if (set_off[s + 1] <= set_off[s])
        return failf(SRS_ERR_INVALID, "binary metrics: set %d is empty or its offsets decrease", s);
  } else if (n_sets != 1) {
    return failf(SRS_ERR_INVALID, "binary metrics: without set offsets n_sets must be 1, got %d", n_sets);
  }
  return SRS_OK;
}

template <class S, class L>
int create(const S* scores, const L* labels, bool on_device, int64_t n64, const int64_t* set_off_in, int32_t n_sets,
           int32_t num_bins, int32_t device, void* stream, srs_binary_metrics** out) {
  PROPAGATE(check_args(scores, labels, n64, set_off_in, n_sets, num_bins, out));
  const int n = (int)n64;
  std::vector<int64_t> set_off(n_sets + 1);
  if (set_off_in) std::memcpy(set_off.data(), set_off_in, sizeof(int64_t) * (n_sets + 1));
  else set_off = {0, n64};

  HostCall c;
  PROPAGATE(c.begin(device));
  const S* d_score = scores;
  const L* d_label = labels;
  if (on_device) {                               // read the inputs after the work queued on the caller's stream
    cudaEvent_t ev;
    CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    cudaError_t e = cudaEventRecord(ev, (cudaStream_t)stream);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(c.s, ev, 0);
    cudaEventDestroy(ev);
    CUDA_TRY(e);
  } else {
    S* ds;
    L* dl;
    PROPAGATE(c.upload(&ds, scores, n));
    PROPAGATE(c.upload(&dl, labels, n));
    d_score = ds;
    d_label = dl;
  }
  int64_t* d_set_off;
  PROPAGATE(c.upload(&d_set_off, set_off.data(), n_sets + 1));

  // keys and the (set, descending score) sort
  uint64_t *k0, *k1;
  uint32_t *t0, *t1;
  CUDA_TRY(c.sc.alloc(&k0, n));
  CUDA_TRY(c.sc.alloc(&k1, n));
  CUDA_TRY(c.sc.alloc(&t0, n));
  CUDA_TRY(c.sc.alloc(&t1, n));
  bm_keys_kernel<<<grid_for(n, 256), 256, 0, c.s>>>(d_score, d_label, n, d_set_off, n_sets, k0, t0);
  LAUNCHED();
  cub::DoubleBuffer<uint64_t> kb(k0, k1);
  cub::DoubleBuffer<uint32_t> tb(t0, t1);
  // A float32 score widened to double has its 29 low mantissa bits zero, so its key's low 29 bits are all ones
  // (sign clear) or all zeros (sign set, or NaN): keys equal in bits 29..63 are equal, and those bits alone sort.
  constexpr int kBeginBit = sizeof(S) == sizeof(float) ? 29 : 0;
  CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, kb, tb, n, kBeginBit, 64, c.s));
  if (n_sets > 1) {
    int bits = 1;
    while (bits < 31 && ((n_sets - 1) >> bits)) ++bits;
    CUB_RUN(c, cub::DeviceRadixSort::SortPairs(tmp__, tb__, tb, kb, n, 1, 1 + bits, c.s));
  }
  const uint64_t* key = kb.Current();

  // runs and cumulative positives
  uint8_t* head;
  int32_t *cum, *run_start;
  int* d_nruns;
  CUDA_TRY(c.sc.alloc(&head, n));
  CUDA_TRY(c.sc.alloc(&cum, n));
  CUDA_TRY(c.sc.alloc(&run_start, n));
  CUDA_TRY(c.sc.alloc(&d_nruns, 1));
  bm_heads_kernel<<<grid_for(n, 256), 256, 0, c.s>>>(key, tb.Current(), n, head, cum);
  LAUNCHED();
  CUB_RUN(c, cub::DeviceScan::InclusiveSum(tmp__, tb__, cum, cum, n, c.s));
  CUB_RUN(c, cub::DeviceSelect::Flagged(tmp__, tb__, thrust::counting_iterator<int32_t>(0), head, run_start,
                                         d_nruns, n, c.s));
  int64_t *d_run_off, *d_pos;
  CUDA_TRY(c.sc.alloc(&d_run_off, n_sets + 1));
  CUDA_TRY(c.sc.alloc(&d_pos, n_sets));
  bm_sets_kernel<<<grid_for(n_sets, 256), 256, 0, c.s>>>(d_set_off, n_sets, run_start, d_nruns, cum, d_run_off,
                                                          d_pos);
  LAUNCHED();
  std::vector<int64_t> run_off(n_sets + 1), pos(n_sets);
  CUDA_TRY(cudaMemcpyAsync(run_off.data(), d_run_off, sizeof(int64_t) * (n_sets + 1), cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(pos.data(), d_pos, sizeof(int64_t) * n_sets, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));

  // binning and the point layout (host): grouping = runs / numBins, none below 2
  std::vector<int64_t> pt_off(n_sets + 1, 0), ch_off(n_sets + 1, 0);
  std::vector<int32_t> grouping(n_sets);
  for (int32_t s = 0; s < n_sets; ++s) {
    const int64_t runs = run_off[s + 1] - run_off[s];
    const int64_t g = num_bins > 0 ? runs / num_bins : 0;
    grouping[s] = g < 2 ? 1 : (int32_t)g;
    const int64_t T = (runs + grouping[s] - 1) / grouping[s];
    pt_off[s + 1] = pt_off[s] + T;
    ch_off[s + 1] = ch_off[s] + (T + kChunk - 1) / kChunk;
  }
  const int64_t n_points = pt_off[n_sets], n_chunks = ch_off[n_sets];
  int64_t *d_pt_off, *d_ch_off;
  int32_t* d_grouping;
  PROPAGATE(c.upload(&d_pt_off, pt_off.data(), n_sets + 1));
  PROPAGATE(c.upload(&d_ch_off, ch_off.data(), n_sets + 1));
  PROPAGATE(c.upload(&d_grouping, grouping.data(), n_sets));

  srs_binary_metrics* h = new (std::nothrow) srs_binary_metrics;
  if (!h) return failf(SRS_ERR_NOMEM, "binary metrics: out of host memory");
  std::unique_ptr<srs_binary_metrics> owner(h);
  h->device = device;
  CUDA_TRY(cudaMalloc(&h->thr, sizeof(double) * n_points));
  CUDA_TRY(cudaMalloc(&h->tp, sizeof(int64_t) * n_points));
  CUDA_TRY(cudaMalloc(&h->fp, sizeof(int64_t) * n_points));
  bm_points_kernel<<<grid_for(n_points, 256), 256, 0, c.s>>>(
      PointArgs{d_pt_off, d_grouping, d_run_off, d_set_off, n_sets}, n_points, run_start, key, cum, h->thr, h->tp,
      h->fp);
  LAUNCHED();

  double *part, *d_area;
  CUDA_TRY(c.sc.alloc(&part, 2 * n_chunks));
  CUDA_TRY(c.sc.alloc(&d_area, 2 * (size_t)n_sets));
  const AreaArgs aa{d_pt_off, d_ch_off, d_pos, d_set_off, n_sets};
  bm_area_chunk_kernel<<<(unsigned)n_chunks, kChunkThreads, 0, c.s>>>(aa, h->tp, h->fp, part, part + n_chunks);
  LAUNCHED();
  bm_area_set_kernel<<<(unsigned)((n_sets + 7) / 8), 256, 0, c.s>>>(aa, h->tp, h->fp, part, part + n_chunks, d_area,
                                                                     d_area + n_sets);
  LAUNCHED();
  h->roc.resize(n_sets);
  h->pr.resize(n_sets);
  CUDA_TRY(cudaMemcpyAsync(h->roc.data(), d_area, sizeof(double) * n_sets, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(h->pr.data(), d_area + n_sets, sizeof(double) * n_sets, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));

  h->n_sets = n_sets;
  h->n.resize(n_sets);
  for (int32_t s = 0; s < n_sets; ++s) h->n[s] = set_off[s + 1] - set_off[s];
  h->positives = std::move(pos);
  h->pt_off = std::move(pt_off);
  *out = owner.release();
  return SRS_OK;
}

int check_set(const srs_binary_metrics* h, int32_t set) {
  if (!h) return failf(SRS_ERR_INVALID, "binary metrics: null handle");
  if (set < 0 || set >= h->n_sets)
    return failf(SRS_ERR_INVALID, "binary metrics: set %d out of range 0 .. %d", set, h->n_sets - 1);
  return SRS_OK;
}

}  // namespace
}  // namespace srs

using namespace srs;

extern "C" int srs_binary_metrics_create_host(const double* scores, const double* labels, int64_t n,
                                              const int64_t* set_off, int32_t n_sets, int32_t num_bins,
                                              int32_t device, srs_binary_metrics** out) {
  return create(scores, labels, false, n, set_off, n_sets, num_bins, device, nullptr, out);
}

extern "C" int srs_binary_metrics_create_device(const float* scores, const int32_t* labels, int64_t n,
                                                const int64_t* set_off, int32_t n_sets, int32_t num_bins,
                                                int32_t device, void* stream, srs_binary_metrics** out) {
  return create(scores, labels, true, n, set_off, n_sets, num_bins, device, stream, out);
}

extern "C" void srs_binary_metrics_destroy(srs_binary_metrics* h) { delete h; }

extern "C" int srs_binary_metrics_summary(const srs_binary_metrics* h, int32_t set, srs_binary_summary* out) {
  PROPAGATE(check_set(h, set));
  if (!out) return failf(SRS_ERR_INVALID, "binary metrics: null summary");
  out->n = h->n[set];
  out->positives = h->positives[set];
  out->negatives = h->n[set] - h->positives[set];
  out->thresholds = h->pt_off[set + 1] - h->pt_off[set];
  out->area_under_roc = h->roc[set];
  out->area_under_pr = h->pr[set];
  return SRS_OK;
}

extern "C" int srs_binary_metrics_curve(const srs_binary_metrics* h, int32_t set, int32_t which, double beta,
                                        double* dst) {
  PROPAGATE(check_set(h, set));
  if (which < SRS_BM_ROC || which > SRS_BM_FMEASURE)
    return failf(SRS_ERR_INVALID, "binary metrics: unknown curve %d", which);
  if (!dst) return failf(SRS_ERR_INVALID, "binary metrics: null destination");
  const int64_t first = h->pt_off[set], T = h->pt_off[set + 1] - first;
  const int64_t len = which == SRS_BM_ROC ? 2 * (T + 2) : which == SRS_BM_PR ? 2 * (T + 1)
                      : which == SRS_BM_THRESHOLDS ? T : 2 * T;
  HostCall c;
  PROPAGATE(c.begin(h->device));
  double* d_out;
  CUDA_TRY(c.sc.alloc(&d_out, len));
  bm_curve_kernel<<<grid_for(len, 256), 256, 0, c.s>>>(which, beta, first, T, h->positives[set],
                                                        h->n[set] - h->positives[set], h->thr, h->tp, h->fp, d_out);
  LAUNCHED();
  CUDA_TRY(cudaMemcpyAsync(dst, d_out, sizeof(double) * len, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));
  return SRS_OK;
}

extern "C" int srs_binary_metrics_confusion(const srs_binary_metrics* h, int32_t set, int64_t* tp, int64_t* fp) {
  PROPAGATE(check_set(h, set));
  if (!tp || !fp) return failf(SRS_ERR_INVALID, "binary metrics: null destination");
  const int64_t first = h->pt_off[set], T = h->pt_off[set + 1] - first;
  HostCall c;
  PROPAGATE(c.begin(h->device));
  CUDA_TRY(cudaMemcpyAsync(tp, h->tp + first, sizeof(int64_t) * T, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaMemcpyAsync(fp, h->fp + first, sizeof(int64_t) * T, cudaMemcpyDeviceToHost, c.s));
  CUDA_TRY(cudaStreamSynchronize(c.s));
  return SRS_OK;
}
