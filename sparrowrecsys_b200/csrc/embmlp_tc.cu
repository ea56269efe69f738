// embmlp_tc.cu - EmbeddingMLP / Wide&Deep forward on the tensor cores (warpgroup MMAs, wgmma) for
// the reference shape (E <= 12: ten 12-float embedding slots = 120 of 128 K columns).
//
// Reference: EmbeddingMLP.py:72-77 and WideNDeep.py:101-107
// (TFRecModel/src/com/sparrowrecsys/offline/tensorflow/).  Both Dense(128) layers are computed
// transposed - D[128 units x rows] = W^T[128 x 128] . X^T - so the 64 rows of a super-group are
// the MMA's N and the weights, resident in shared memory as bf16 hi/lo images, its M (warpgroup
// q issues units 64 q .. 64 q + 63).  Operands are split x = hi + lo (bf16x3: hi*hi + lo*hi +
// hi*lo, fp32 accumulate); the activations' hi and lo halves are stacked along N ([64 rows hi |
// 64 rows lo]), so a layer is 8 K steps x 2 MMAs of m64n128k16 per warpgroup.  The 7 raw-scale
// numerics never enter an MMA: their contribution is added in fp32 in the layer-1 epilogue.
//
// One persistent CTA per SM, 256 threads; per super-group of 64 rows: 30 row gathers per row
// straight into the X operand tile, MMAs, epilogue on the accumulator registers (thread = 2
// units x 16 rows) -> H1 operand tile over the X tile, MMAs, epilogue, Dense(1) (+ the W&D
// wide weight), sigmoid.
#include "kernels.h"
#include "wgmma.cuh"

namespace srs {
using namespace wg;

constexpr int kEtRows = 64;                              // rows per super-group = half of the MMA N
// shared-memory image: four 32 KB operands, each 2 K blocks x [128 units][64 k] bf16 SW128
constexpr uint32_t EIMG_W1_HI = 0, EIMG_W1_LO = 32768, EIMG_W2_HI = 65536, EIMG_W2_LO = 98304;
constexpr uint32_t EIMG_BYTES = 131072;
// scratch
constexpr uint32_t ES_X = 0;                             // 2 K blocks x [64 hi | 64 lo rows][64 k] = 32 KB
constexpr uint32_t ES_RED = 32768;                       // f32 [128 units][64 rows] = 32 KB
constexpr uint32_t ES_NUMS = 65536;                      // f32 [64][8]
constexpr uint32_t ES_ZP = 67584;                        // f32 [4][64]
constexpr uint32_t ES_BYTES = 68608;

__global__ void __launch_bounds__(256, 1) embmlp_tc_kernel(const __grid_constant__ EmbMlpParams p,
                                                            BatchView b) {
  extern __shared__ uint8_t raw[];
  __shared__ uint64_t wbar;
  __shared__ float b3;      // dense_2/bias from the blob, once per CTA (a register would stay live through the MMAs)
  const int tid = threadIdx.x, q = tid >> 7, tw = tid & 127, warp_w = tw >> 5;
  const int lane = tw & 31, g = lane >> 2, cq = lane & 3;
  uint8_t* base = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
  uint8_t* img = base;
  uint8_t* sc = base + EIMG_BYTES;
  float* nums = reinterpret_cast<float*>(sc + ES_NUMS);
  float* red = reinterpret_cast<float*>(sc + ES_RED);
  float* zp = reinterpret_cast<float*>(sc + ES_ZP);

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (tid == 0) {
    mbar_init(&wbar, 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(&wbar, EIMG_BYTES);
    for (uint32_t off = 0; off < EIMG_BYTES; off += 32768u) bulk_g2s(img + off, p.image + off, 32768u, &wbar);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  __syncthreads();
  const uint32_t s_img = smem_u32(img), s_x = smem_u32(sc + ES_X);
  bool weights_ready = false;
  // the numerics' rows of W1 (EmbMlpBlob at EP = 12: rows 120..127, after the ten slots), which no MMA takes
  const float* w1_numerics = p.W1 + 10 * 12 * 128;
  // this thread's accumulator rows are units u_i = 64 q + 16 warp_w + g + 8 i of both layers
  float b1[2], b2[2], w3[2], w1n[2][kNumNumerics];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int u = 64 * q + 16 * warp_w + g + 8 * i;
    b1[i] = __ldg(p.b1 + u); b2[i] = __ldg(p.b2 + u); w3[i] = __ldg(p.w3 + u);
#pragma unroll
    for (int n = 0; n < kNumNumerics; ++n) w1n[i][n] = __ldg(w1_numerics + n * 128 + u);
  }
  if (tid == 0) b3 = __ldg(p.b3);                        // the layers' barriers order it before the Dense(1)

  const int n_sg = (b.B + kEtRows - 1) / kEtRows;
  for (int sg = blockIdx.x; sg < n_sg; sg += gridDim.x) {
    const int row0 = sg * kEtRows;
    // ---- gathers -> X operand tile (K = slot * 12 + e; columns 120..127 are zero) ---------
    for (int i = tid; i < kEtRows * 32; i += 256) {      // 64 rows x 32 float4 (30 gathered + 2 zero)
      const int r = i >> 5, f = i & 31;
      const int row = row0 + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < 30 && row < b.B) {
        const int slot = f / 3, q = f - slot * 3;
        int id;
        const float* table;
        if (slot < 3) {
          id = __ldg(b.movie_genre + row * 3 + slot);
          table = p.genre[slot];
        } else if (slot == 3) {
          id = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
          table = p.movie;
        } else if (slot < 9) {
          id = __ldg(b.user_genre + row * 5 + (slot - 4));
          table = p.genre[slot - 1];
        } else {
          id = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
          table = p.user;
        }
        if (slot != 3 && slot != 9) {
          if (id >= p.n_genres) { atomicExch(b.err_flag, 1); id = -1; }
        }
        if (id >= 0) v = ldg4(table + (size_t)id * 12 + 4 * q);
      }
      const int k = 4 * f;                               // K index of v.x (slot*12 + 4q == 4f)
      const uint32_t off = (uint32_t)(k >> 6) * 16384u + sw128_offset(r, (k & 63) >> 3) + ((k & 4) ? 8u : 0u);
      const Split2 s0 = split_pack(v.x, v.y), s1 = split_pack(v.z, v.w);
      *reinterpret_cast<uint2*>(sc + ES_X + off) = make_uint2(s0.hi, s1.hi);
      *reinterpret_cast<uint2*>(sc + ES_X + off + 8192u) = make_uint2(s0.lo, s1.lo);   // row + 64
    }
    for (int i = tid; i < kEtRows * 8; i += 256) {
      const int r = i >> 3, j = i & 7;
      const int row = row0 + r;
      nums[i] = (j < kNumNumerics && row < b.B) ? __ldg(b.numerics + row * kNumNumerics + j) : 0.f;
    }
    fence_async_smem();
    __syncthreads();
    if (!weights_ready) { mbar_wait(&wbar, 0); weights_ready = true; }

    // ---- two Dense(128, relu) layers ----------------------------------------------------
#pragma unroll 1
    for (int layer = 0; layer < 2; ++layer) {
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0.f;
      {
        const uint32_t a_hi = s_img + (layer == 0 ? EIMG_W1_HI : EIMG_W2_HI) + q * 8192;   // units 64 q ..
        const uint32_t a_lo = s_img + (layer == 0 ? EIMG_W1_LO : EIMG_W2_LO) + q * 8192;
        mma_fence();
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
          const uint64_t ah = desc_sw128(a_hi + kb * 16384), al = desc_sw128(a_lo + kb * 16384);
          const uint64_t xs = desc_sw128(s_x + kb * 16384);                 // [X hi | X lo], N = 128
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            mma_m64n128_ss(d, ah + 2 * ks, xs + 2 * ks, kb > 0 || ks > 0);
            mma_m64n128_ss(d, al + 2 * ks, xs + 2 * ks, 1);
          }
        }
        mma_commit();
        mma_wait<0>();
        reg_fence(d);
      }
      __syncthreads();                                     // both warpgroups' MMAs have read X
      // epilogue: units u_i, rows r = 8 j + 2 cq + c (X hi: column r, X lo: column 64 + r)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int u = 64 * q + 16 * warp_w + g + 8 * i;
        const uint32_t koff = (uint32_t)(u >> 6) * 16384u, chunk = (u & 63) >> 3, within = (u & 7) * 2;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int r = 8 * j + 2 * cq + c;
            float v = d[4 * j + 2 * i + c] + d[4 * (j + 8) + 2 * i + c];
            if (layer == 0) {
              const float4 n0 = *reinterpret_cast<const float4*>(nums + r * 8);
              const float4 n1 = *reinterpret_cast<const float4*>(nums + r * 8 + 4);
              v += b1[i];
              v = fmaf(n0.x, w1n[i][0], v); v = fmaf(n0.y, w1n[i][1], v); v = fmaf(n0.z, w1n[i][2], v);
              v = fmaf(n0.w, w1n[i][3], v); v = fmaf(n1.x, w1n[i][4], v); v = fmaf(n1.y, w1n[i][5], v);
              v = fmaf(n1.z, w1n[i][6], v);
              v = fmaxf(v, 0.f);
              const uint32_t off = koff + sw128_offset(r, chunk) + within;   // H1[row r][k = unit u]
              const __nv_bfloat16 vh = __float2bfloat16_rn(v);
              *reinterpret_cast<__nv_bfloat16*>(sc + ES_X + off) = vh;
              *reinterpret_cast<__nv_bfloat16*>(sc + ES_X + off + 8192u) = __float2bfloat16_rn(v - __bfloat162float(vh));
            } else {
              red[u * kEtRows + r] = fmaxf(v + b2[i], 0.f) * w3[i];
            }
          }
      }
      fence_async_smem();
      __syncthreads();
    }
    // ---- Dense(1): sum over the 128 units, + wide weight (W&D), sigmoid ------------------------
    {
      const int r = tid & 63, part = tid >> 6;             // 4 parts x 32 units
      float s = 0.f;
#pragma unroll 8
      for (int u = 0; u < 32; ++u) s += red[(part * 32 + u) * kEtRows + r];
      zp[part * kEtRows + r] = s;
    }
    __syncthreads();
    if (tid < kEtRows) {
      const int row = row0 + tid;
      if (row < b.B) {
        float z = b3 + ((zp[tid] + zp[kEtRows + tid]) + (zp[2 * kEtRows + tid] + zp[3 * kEtRows + tid]));
        if (p.wide) {
          const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
          const int rated = checked_id(__ldg(b.hist + (size_t)row * b.hist_stride), p.n_movies, b.err_flag);
          z += __ldg(p.wide + crossed_bucket(mid, rated, (uint32_t)p.cross_buckets));
        }
        store_score(b, row, sigmoidf_acc(z));
        if (b.logits) b.logits[row] = z;
      }
    }
    __syncthreads();
  }
  if (!weights_ready) mbar_wait(&wbar, 0);
}

static size_t embmlp_tc_smem() { return 1024 + EIMG_BYTES + ES_BYTES; }

cudaError_t launch_embmlp_tc(const EmbMlpParams& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  const int n_sg = (b.B + kEtRows - 1) / kEtRows;
  const int grid = n_sg < p.num_sms ? n_sg : p.num_sms;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = embmlp_tc_smem();
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  ++g_launch_count;
  return cudaLaunchKernelEx(&cfg, embmlp_tc_kernel, p, b);
}

cudaError_t setup_embmlp_tc_attributes() {
  return cudaFuncSetAttribute(embmlp_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)embmlp_tc_smem());
}

}  // namespace srs
