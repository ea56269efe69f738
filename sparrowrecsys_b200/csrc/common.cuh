// common.cuh - device helpers shared by the fused CTR forward kernels (sm_90a).
//
// The kernels restate the reference graphs
// (TFRecModel/src/com/sparrowrecsys/offline/tensorflow/*.py) on a private device
// layout: embedding tables padded to EP = round-up(E, 4) floats per row so every
// row gather is a run of aligned 128-bit loads, first Dense kernels permuted to the
// order the kernel stages its input tile in (embedding slots first, numerics last),
// hidden widths zero-padded.  model.cu builds that layout; nothing here is visible
// at the C ABI.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace srs {

constexpr int kThreads = 256;          // every tile kernel runs 8 warps per CTA
constexpr int kNumNumerics = 7;
constexpr int kNumPad = 8;             // numerics padded to 8 floats in the input tile

enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_PRELU = 2 };

// ---- batch view (device pointers) ------------------------------------------------
struct BatchView {
  int B;
  int hist_stride;
  const int32_t* movie_id;
  const int32_t* user_id;
  const int32_t* hist;
  const int32_t* movie_genre;   // [B,3]
  const int32_t* user_genre;    // [B,5]
  const float* numerics;        // [B,7]
  float* probs;                 // [B]
  float* logits;                // [B] or nullptr
  int* err_flag;                // latched when an id is out of range
  // ---- score exchange of a ranking call that spans GPUs (gather.cu; all zero otherwise) ----------
  // `probs` is then this rank's slice of its own gather buffer and peer_probs[k] the same slice of
  // the other ranks' buffers (peer memory over NVLink): the epilogue stores each score N times and
  // no collective follows.  Kernels that end with gather_signal_tail() also publish the step number
  // to every rank's flag word once their last CTA has finished.
  float* peer_probs[7];
  int n_peers;
  int n_sig;                    // ranks to signal (0: no in-kernel signal)
  uint32_t* sig_flags[8];       // flag word of THIS rank in every rank's flag array (own included)
  unsigned int* sig_counter;    // local: [0] CTAs of this launch that have finished, [1] steps signalled so far (the
                                // step number lives on the device so that a captured CUDA graph can be replayed)
};

__device__ __forceinline__ void store_score(const BatchView& b, int row, float v) {
  b.probs[row] = v;
  for (int k = 0; k < b.n_peers; ++k) b.peer_probs[k][row] = v;
}

// Last statement of a kernel that supports the in-kernel signal (every thread calls it): when the
// last CTA of the launch gets here, every score of this rank's slice has been stored - locally and
// on the peers - and the step number goes out to the flag words the waiters poll.
__device__ __forceinline__ void gather_signal_tail(const BatchView& b) {
  if (b.n_sig == 0) return;
  __syncthreads();                           // the CTA's score stores happen-before this barrier ...
  if (threadIdx.x == 0) {
    __threadfence_system();                  // ... and one cumulative system-scope fence publishes them (a fence in
                                             // every thread cost ~10 us per launch over NVLink)
    const unsigned int done = atomicAdd(b.sig_counter, 1u) + 1u;
    if (done == gridDim.x) {
      b.sig_counter[0] = 0u;
      const uint32_t step = ++b.sig_counter[1];
      __threadfence_system();
      for (int k = 0; k < b.n_sig; ++k) *reinterpret_cast<volatile uint32_t*>(b.sig_flags[k]) = step;
    }
  }
}

// ---- opt-in phase timing of the DIN kernels (tools/din_phases.py builds the library with -DSRS_DIN_PHASES) ----
// One lead thread per timing unit (a warpgroup of din_wg_kernel, warp 0 of din_kernel) adds the clock64()
// cycles since its previous lap to g_din_phases[phase]; in the default build a lap compiles to nothing.
enum DinPhase {
  PH_TILE_INPUTS = 0,   // side features, candidate rows, activation-unit constants
  PH_W_BUILD,           // per-row B operand W_r (wgmma) / folded column (CUDA cores)
  PH_GATHER_ISSUE,      // history ids and history-row gathers issued
  PH_GATHER_WAIT,       // waiting for the gathers of the current row
  PH_AU_MMA,            // activation-unit MMAs, issue to completion
  PH_GATE,              // PReLU, Dense(1), sigmoid per position
  PH_POOL,              // weighted sum of the history rows
  PH_AU_LOOP,           // CUDA-core kernel: activation unit + gate + pooling per position
  PH_ROW_IMBALANCE,     // waiting at the barrier before the top MLP
  PH_TOP_MLP,           // Dense(128) / Dense(64) / Dense(1) + sigmoid
  PH_IMAGE_WAIT,        // waiting for the top-MLP weight image (din_wg_kernel, E <= 32)
  kDinPhases
};
#ifdef SRS_DIN_PHASES
static __device__ unsigned long long g_din_phases[kDinPhases];
struct PhaseClock {
  long long t = 0;
  bool lead;
  __device__ explicit PhaseClock(bool lead_) : lead(lead_) {
#ifdef __CUDA_ARCH__
    t = clock64();
#endif
  }
  __device__ void lap(int ph) {
#ifdef __CUDA_ARCH__
    const long long n = clock64();
    if (lead) atomicAdd(&g_din_phases[ph], (unsigned long long)(n - t));
    t = n;
#endif
  }
};
// copy the counters of this translation unit's kernel to the host and clear them
static inline cudaError_t din_phases_take(unsigned long long* out) {
  cudaError_t e = cudaMemcpyFromSymbol(out, g_din_phases, sizeof(unsigned long long) * kDinPhases);
  if (e != cudaSuccess) return e;
  static const unsigned long long zero[kDinPhases] = {};
  return cudaMemcpyToSymbol(g_din_phases, zero, sizeof zero);
}
#else
struct PhaseClock {
  __device__ explicit PhaseClock(bool) {}
  __device__ void lap(int) {}
};
#endif

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

__device__ __forceinline__ float sigmoidf_acc(float x) {
  // 1/(1+e^-x) the way the oracle evaluates it (stable on both sides)
  if (x >= 0.f) return 1.f / (1.f + expf(-x));
  float e = expf(x);
  return e / (1.f + e);
}

// Keras's binary_crossentropy of one row of a sigmoid output layer in float32: the logit path
// max(x, 0) - x*z + log1p(exp(-|x|)) (sigmoid_cross_entropy_with_logits), label z in {0, 1}
__device__ __forceinline__ float logit_bce(float x, int z) {
  const float relu = fmaxf(x, 0.f);
  const float xz = z ? x : 0.f;                    // x * z, z in {0, 1}
  return __fadd_rn(__fsub_rn(relu, xz), log1pf(expf(-fabsf(x))));
}

// A training step's dL/dz for a row of a batch of B with weight w: (w (p - y)) / B (Keras's SUM_OVER_BATCH_SIZE: the
// denominator is B, not the weights' sum), and (p - y) / B when not `weighted`.  w = 1 gives the unweighted bits.
__device__ __forceinline__ float row_dz(float p, int y, bool weighted, float w, int B) {
  const float g = __fsub_rn(p, (float)y);
  return __fdiv_rn(weighted ? __fmul_rn(w, g) : g, (float)B);
}
// the same with w = weight[row], weight null: unweighted
__device__ __forceinline__ float row_dz(float p, int y, const float* weight, int row, int B) {
  return row_dz(p, y, weight != nullptr, weight ? __ldg(weight + row) : 1.f, B);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// id range check mirroring categorical_column_with_identity's asserts: an
// out-of-range id latches the error flag and is read as row 0 (never faults).
__device__ __forceinline__ int checked_id(int id, int limit, int* err_flag) {
  if (static_cast<unsigned>(id) >= static_cast<unsigned>(limit)) {
    if (err_flag) atomicExch(err_flag, 1);
    return 0;
  }
  return id;
}

// ---- tile MLP on CUDA cores -----------------------------------------------------
// ys[r][n] = act( sum_k xs[r][k] * W[k][n] + bias[n] )   r < R, n < N
//   xs : shared, row-major, leading dim ldx (multiple of 4 floats), K multiple of 4
//   W  : global, row-major [K][N] (weights are tiny and shared by every CTA: they
//        stay L1/L2 resident, so they are read through the read-only path rather
//        than staged)
// Thread (cx, ry) owns TM rows x TN columns; lanes of a warp sweep the columns so W
// loads are contiguous 128-bit loads and xs loads are broadcasts.
// W_SMEM: W points into shared memory (staged by stage_weights below) instead of global.
template <int R, int N, int TM, int TN, bool W_SMEM = false>
__device__ __forceinline__ void dense_layer(const float* __restrict__ xs, int ldx, int K,
                                            const float* __restrict__ W,
                                            const float* __restrict__ bias, int act,
                                            const float* __restrict__ alpha,
                                            float* __restrict__ ys, int ldy) {
  constexpr int CT = N / TN;            // column threads
  constexpr int RT = kThreads / CT;     // row threads
  static_assert(N % TN == 0 && kThreads % CT == 0, "bad column tiling");
  static_assert(RT * TM == R, "row tiling must cover the tile exactly");
  static_assert(TN % 4 == 0, "TN must be a multiple of 4");
  const int cx = threadIdx.x % CT;
  const int ry = threadIdx.x / CT;
  const int col0 = cx * TN;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  // weights stream from L2/L1: the next 4 rows of W are requested before the current 4 are used
  float4 wn[4][TN / 4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int j = 0; j < TN / 4; ++j)
      wn[kk][j] = W_SMEM ? *reinterpret_cast<const float4*>(W + (size_t)kk * N + col0 + 4 * j)
                         : ldg4(W + (size_t)kk * N + col0 + 4 * j);
  for (int k = 0; k < K; k += 4) {
    float4 xv[TM];
    float4 wc[4][TN / 4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int j = 0; j < TN / 4; ++j) wc[kk][j] = wn[kk][j];
    if (k + 4 < K) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int j = 0; j < TN / 4; ++j)
          wn[kk][j] = W_SMEM ? *reinterpret_cast<const float4*>(W + (size_t)(k + 4 + kk) * N + col0 + 4 * j)
                             : ldg4(W + (size_t)(k + 4 + kk) * N + col0 + 4 * j);
    }
#pragma unroll
    for (int i = 0; i < TM; ++i)
      xv[i] = *reinterpret_cast<const float4*>(xs + (ry + i * RT) * ldx + k);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      float w[TN];
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const float4 t = wc[kk][j / 4];
        w[j] = t.x; w[j + 1] = t.y; w[j + 2] = t.z; w[j + 3] = t.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i) {
        const float x = kk == 0 ? xv[i].x : kk == 1 ? xv[i].y : kk == 2 ? xv[i].z : xv[i].w;
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(x, w[j], acc[i][j]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int r = ry + i * RT;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      float v = acc[i][j] + __ldg(bias + col0 + j);
      if (act == ACT_RELU) v = fmaxf(v, 0.f);
      else if (act == ACT_PRELU) v = v > 0.f ? v : __ldg(alpha + col0 + j) * v;
      ys[r * ldy + col0 + j] = v;
    }
  }
}

// Asynchronous global -> shared copy of a dense weight array (floats multiple of 4, 16-byte
// aligned both sides) by the whole CTA: the per-K-step L2 latency of reading weights in place
// becomes one bulk latency that overlaps the embedding gathers.  Pair with stage_wait().  NT: the
// CTA's thread count.
template <int NT = kThreads>
__device__ __forceinline__ void stage_weights(float* dst_smem, const float* __restrict__ src, int n_floats) {
  const uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(dst_smem));
  for (int i = threadIdx.x * 4; i < n_floats; i += NT * 4)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + i * 4), "l"(src + i) : "memory");
}
__device__ __forceinline__ void stage_wait() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

// z[r] = sum_k xs[r][k] * w[k]   one warp per row, rows strided over the 8 warps.
template <int R, typename F>
__device__ __forceinline__ void row_dot(const float* __restrict__ xs, int ldx, int K,
                                        const float* __restrict__ w, F&& emit) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < R; r += kThreads / 32) {
    float s = 0.f;
    for (int k = lane; k < K; k += 32) s = fmaf(xs[r * ldx + k], __ldg(w + k), s);
    s = warp_sum(s);
    if (lane == 0) emit(r, s);
  }
}

// Cooperative gather of one embedding row per (tile row, slot) into the input tile.
//   item i in [0, R*Q): row = i / Q, q = i % Q, copies floats [4q, 4q+4) of table row id.
template <int EP>
__device__ __forceinline__ void gather_row(float* dst, const float* __restrict__ table,
                                           int id /* -1 = zero vector */, int q) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (id >= 0) v = ldg4(table + (size_t)id * EP + 4 * q);
  *reinterpret_cast<float4*>(dst + 4 * q) = v;
}

// Side features of a 32-row tile shared by the DIN-family kernels: the userGenre1, userId and
// movieGenre1 embedding rows (DenseFeatures columns of the user-profile / context layers, e.g.
// DIN.py:108-123) land at tile columns off_ug / off_u / off_mg, the 7 numerics (+ one zero pad) at
// off_num.  Rows past the batch end and missing / OOV genres (-1) are zero; an id outside its
// vocabulary latches the error flag.  The ids are read here, the rows and numerics are copied by
// cp.async (16-byte row chunks, 4-byte numerics, a zero fill where the row is zero) that is not
// waited for: the caller waits for its cp.async groups (stage_wait) and passes a barrier before
// the tile is read.  NT: the CTA's thread count.  kRowsL1: the rows are copied through L1 (cp.async.ca), which
// din_wg_kernel wants (its gathers keep L1 for rows, and the 20 genre rows recur in every tile), instead of L2
// only (.cg), which measured about 1 % faster for din_kernel.  Valid because no predict launch writes a table
// that it gathers (L1 does not see other SMs' writes).
template <int EP, int R, int NT = kThreads, bool kRowsL1 = false>
__device__ __forceinline__ void tile_side_features(float* __restrict__ Xs, int ldx, int row0,
                                                   const BatchView& b, const float* user,
                                                   const float* ugenre, const float* mgenre,
                                                   int n_users, int n_genres, int off_ug, int off_u,
                                                   int off_mg, int off_num) {
  constexpr int Q = EP / 4;
  const uint32_t xs = static_cast<uint32_t>(__cvta_generic_to_shared(Xs));
  for (int i = threadIdx.x; i < R * 3 * Q; i += NT) {
    const int q = i % Q;
    const int t = i / Q;
    const int slot = t % 3;
    const int r = t / 3;
    const int row = row0 + r;
    int id = -1;
    const float* table = user;
    const int off = slot == 0 ? off_ug : slot == 1 ? off_u : off_mg;
    if (row < b.B) {
      if (slot == 1) {
        id = checked_id(__ldg(b.user_id + row), n_users, b.err_flag);
      } else {
        id = slot == 0 ? __ldg(b.user_genre + row * 5) : __ldg(b.movie_genre + row * 3);
        if (id >= n_genres) { atomicExch(b.err_flag, 1); id = -1; }
        if (id < 0) id = -1;
        table = slot == 0 ? ugenre : mgenre;
      }
    }
    // source size 0 reads nothing (the address stays a valid row) and zero-fills the 16 bytes
    if constexpr (kRowsL1)
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;"
                   ::"r"(xs + 4u * (r * ldx + off + 4 * q)), "l"(table + (size_t)max(id, 0) * EP + 4 * q),
                   "r"(id >= 0 ? 16u : 0u) : "memory");
    else
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;"
                   ::"r"(xs + 4u * (r * ldx + off + 4 * q)), "l"(table + (size_t)max(id, 0) * EP + 4 * q),
                   "r"(id >= 0 ? 16u : 0u) : "memory");
  }
  for (int i = threadIdx.x; i < R * kNumPad; i += NT) {
    const int r = i / kNumPad, j = i % kNumPad;
    const int row = row0 + r;
    if (j < kNumNumerics) {
      const bool in = row < b.B;
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;"
                   ::"r"(xs + 4u * (r * ldx + off_num + j)), "l"(b.numerics + (in ? row * kNumNumerics + j : 0)),
                   "r"(in ? 4u : 0u) : "memory");
    } else {
      Xs[r * ldx + off_num + j] = 0.f;
    }
  }
}

// FingerprintCat64 / crossed_column bucket (WideNDeep.py:72-73; restated from
// tensorflow/core/platform/fingerprint.h as recorded in SURVEY.md section 8a row a3).
__host__ __device__ __forceinline__ uint64_t shift_mix(uint64_t v) { return v ^ (v >> 47); }
__host__ __device__ __forceinline__ uint64_t fingerprint_cat64(uint64_t fp1, uint64_t fp2) {
  const uint64_t kMul = 0xc6a4a7935bd1e995ULL;
  uint64_t result = fp1 ^ kMul;
  result ^= shift_mix(fp2 * kMul) * kMul;
  result *= kMul;
  result = shift_mix(result) * kMul;
  result = shift_mix(result);
  return result;
}
__host__ __device__ __forceinline__ uint32_t crossed_bucket(int32_t movie_id, int32_t rated,
                                                            uint32_t buckets) {
  uint64_t h = fingerprint_cat64(0xDECAFCAFFEULL, (uint64_t)(int64_t)movie_id);
  h = fingerprint_cat64(h, (uint64_t)(int64_t)rated);
  return (uint32_t)(h % buckets);
}

}  // namespace srs
