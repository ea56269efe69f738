// deepfm_tc.cu - DeepFM forward with the deep MLP on the tensor cores (warpgroup MMAs), for
// emb_dim 13..16 (EP = 16; BASELINE cfg 2: E = 16, ML-20M vocabularies).
//
// Reference: TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DeepFM.py:91-113.
//   first order : four scalar gathers W[offset + id] (the one-hot x Dense(1) product)
//   FM          : four embedding dots <item,user> <ig,ug> <ig,user> <item,ug>  (CUDA cores)
//   deep        : [deep_item | deep_user | 7 numerics] -> Dense64-relu -> Dense64-relu
// The two Dense(64) layers are computed transposed, D[units x rows] = W^T . X^T, with the 32
// rows of a CTA's super-group as the MMA's N (activations hi/lo stacked along N -> m64n64k16)
// and the 64 units (bf16 hi/lo weight images resident in shared memory) as its M - same scheme
// and same bf16x3 precision as embmlp_tc.cu; the raw-scale numerics stay in fp32.  The CTA is
// one warpgroup.
#include "kernels.h"
#include "wgmma.cuh"

namespace srs {
using namespace wg;

constexpr int kFtRows = 32;                              // rows per super-group
// shared-memory image: [128 (64 used) units][64 k] bf16 SW128 tiles, 16 KB each (layout shared with
// model.cu's image builder; rows 64..127 are zero and not read)
constexpr uint32_t FIMG_W1_HI = 0, FIMG_W1_LO = 16384, FIMG_W2_HI = 32768, FIMG_W2_LO = 49152;
constexpr uint32_t FIMG_BYTES = 65536;
// scratch
constexpr uint32_t FS_X = 0;                             // [32 hi | 32 lo rows][64 k] = 8 KB
constexpr uint32_t FS_F = 8192;                          // f32 [32][4*16 + 4] fm rows = 8704 B
constexpr uint32_t FS_RED = 17408;                       // f32 [64 units][32 rows] = 8 KB
constexpr uint32_t FS_NUMS = 25600;                      // f32 [32][8]
constexpr uint32_t FS_DOTS = 26624;                      // f32 [32][4]
constexpr uint32_t FS_ZP = 27136;                        // f32 [4][32]
constexpr uint32_t FS_BYTES = 27648;

__global__ void __launch_bounds__(128) deepfm_tc_kernel(const __grid_constant__ DeepFmParams p,
                                                        BatchView b) {
  extern __shared__ uint8_t raw[];
  __shared__ uint64_t wbar;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, cq = lane & 3;
  uint8_t* base = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
  uint8_t* img = base;
  uint8_t* sc = base + FIMG_BYTES;
  constexpr int LDF = 4 * 16 + 4;
  float* Fs = reinterpret_cast<float*>(sc + FS_F);
  float* red = reinterpret_cast<float*>(sc + FS_RED);
  float* nums = reinterpret_cast<float*>(sc + FS_NUMS);
  float* dots = reinterpret_cast<float*>(sc + FS_DOTS);
  float* zp = reinterpret_cast<float*>(sc + FS_ZP);

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (tid == 0) {
    mbar_init(&wbar, 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(&wbar, FIMG_BYTES);
    bulk_g2s(img, p.image, 32768u, &wbar);
    bulk_g2s(img + 32768u, p.image + 32768u, 32768u, &wbar);
  }
  // the K padding of the X operand (columns 32..63, hi and lo) is written once
  for (int i = tid; i < 2 * kFtRows * 4; i += 128) {
    const int r = i >> 2, ch = 4 + (i & 3);              // r in 0..63 covers hi rows and lo rows
    *reinterpret_cast<uint4*>(sc + FS_X + sw128_offset(r, ch)) = make_uint4(0, 0, 0, 0);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  __syncthreads();
  const uint32_t s_img = smem_u32(img), s_x = smem_u32(sc + FS_X);
  bool weights_ready = false;
  // the numerics' rows of W1 (DeepFmBlob at EP = 16: rows 32..39, after the deep pair), which no MMA takes
  const float* w1_numerics = p.W1 + 2 * 16 * 64;
  // this thread's accumulator rows are units u_i = 16 warp + g + 8 i of both layers
  float b1[2], b2[2], wdeep[2], w1n[2][kNumNumerics];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int u = 16 * warp + g + 8 * i;
    b1[i] = __ldg(p.b1 + u); b2[i] = __ldg(p.b2 + u); wdeep[i] = __ldg(p.wdeep + u);
#pragma unroll
    for (int n = 0; n < kNumNumerics; ++n) w1n[i][n] = __ldg(w1_numerics + n * 64 + u);
  }

  const int n_sg = (b.B + kFtRows - 1) / kFtRows;
  for (int sg = blockIdx.x; sg < n_sg; sg += gridDim.x) {
    const int row0 = sg * kFtRows;
    // ---- gathers: 6 embedding rows per row; the deep pair goes to the X operand ------------
    for (int i = tid; i < kFtRows * 6 * 4; i += 128) {
      const int q = i & 3, t = i >> 2, slot = t % 6, r = t / 6;
      const int row = row0 + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < b.B) {
        const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
        const int uid = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
        int id;
        const float* table;
        switch (slot) {
          case 0: id = mid; table = p.fm_movie; break;
          case 1: id = uid; table = p.fm_user; break;
          case 2: id = __ldg(b.movie_genre + row * 3); table = p.fm_mgenre; break;
          case 3: id = __ldg(b.user_genre + row * 5); table = p.fm_ugenre; break;
          case 4: id = mid; table = p.deep_movie; break;
          default: id = uid; table = p.deep_user; break;
        }
        if (slot == 2 || slot == 3) {
          if (id >= p.n_genres) { atomicExch(b.err_flag, 1); id = -1; }
        }
        if (id >= 0) v = ldg4(table + (size_t)id * 16 + 4 * q);
      }
      if (slot < 4) {
        *reinterpret_cast<float4*>(Fs + r * LDF + slot * 16 + 4 * q) = v;
      } else {
        const int k = (slot - 4) * 16 + 4 * q;             // K index of v.x
        const uint32_t off = sw128_offset(r, k >> 3) + ((k & 4) ? 8u : 0u);
        const Split2 s0 = split_pack(v.x, v.y), s1 = split_pack(v.z, v.w);
        *reinterpret_cast<uint2*>(sc + FS_X + off) = make_uint2(s0.hi, s1.hi);
        *reinterpret_cast<uint2*>(sc + FS_X + off + 4096u) = make_uint2(s0.lo, s1.lo);   // row + 32
      }
    }
    for (int i = tid; i < kFtRows * 8; i += 128) {
      const int r = i >> 3, j = i & 7;
      const int row = row0 + r;
      nums[i] = (j < kNumNumerics && row < b.B) ? __ldg(b.numerics + row * kNumNumerics + j) : 0.f;
    }
    fence_async_smem();
    __syncthreads();
    if (!weights_ready) { mbar_wait(&wbar, 0); weights_ready = true; }

    // ---- layer 1: K = 32 (two K steps) ----------------------------------------------------------
    float d[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
    {
      const uint64_t ah = desc_sw128(s_img + FIMG_W1_HI), al = desc_sw128(s_img + FIMG_W1_LO);
      const uint64_t xs = desc_sw128(s_x);                                   // [X hi | X lo], N = 64
      mma_fence();
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        mma_m64n64_ss(d, ah + 2 * ks, xs + 2 * ks, ks > 0);
        mma_m64n64_ss(d, al + 2 * ks, xs + 2 * ks, 1);
      }
      mma_commit();
    }
    {  // FM dots while the MMAs run (DeepFM.py:100-103): <item,user> <ig,ug> <ig,user> <item,ug>
      const int r = tid >> 2, dd = tid & 3;
      const float* f = Fs + r * LDF;
      const float* a = (dd == 0 || dd == 3) ? f : f + 32;                    // item or item_genre
      const float* c = (dd == 0 || dd == 2) ? f + 16 : f + 48;               // user or user_genre
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 16; ++k) s = fmaf(a[k], c[k], s);
      dots[tid] = s;
    }
    mma_wait<0>();
    reg_fence(d);
    __syncthreads();                                     // every warp's MMAs have read X
    // epilogue: units u_i, rows r = 8 j + 2 cq + c (X hi: column r, X lo: column 32 + r) -> H1[r][k = u_i]
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int u = 16 * warp + g + 8 * i;
      const uint32_t chunk = u >> 3, within = (u & 7) * 2;
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int r = 8 * j + 2 * cq + c;
          const float4 n0 = *reinterpret_cast<const float4*>(nums + r * 8);
          const float4 n1 = *reinterpret_cast<const float4*>(nums + r * 8 + 4);
          float v = (d[4 * j + 2 * i + c] + d[4 * (j + 4) + 2 * i + c]) + b1[i];
          v = fmaf(n0.x, w1n[i][0], v); v = fmaf(n0.y, w1n[i][1], v); v = fmaf(n0.z, w1n[i][2], v);
          v = fmaf(n0.w, w1n[i][3], v); v = fmaf(n1.x, w1n[i][4], v); v = fmaf(n1.y, w1n[i][5], v);
          v = fmaf(n1.z, w1n[i][6], v);
          v = fmaxf(v, 0.f);
          const uint32_t off = sw128_offset(r, chunk) + within;
          const __nv_bfloat16 vh = __float2bfloat16_rn(v);
          *reinterpret_cast<__nv_bfloat16*>(sc + FS_X + off) = vh;
          *reinterpret_cast<__nv_bfloat16*>(sc + FS_X + off + 4096u) = __float2bfloat16_rn(v - __bfloat162float(vh));
        }
    }
    fence_async_smem();
    __syncthreads();
    // ---- layer 2: K = 64 ----------------------------------------------------------------------------
    {
      const uint64_t ah = desc_sw128(s_img + FIMG_W2_HI), al = desc_sw128(s_img + FIMG_W2_LO);
      const uint64_t hs = desc_sw128(s_x);
      mma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        mma_m64n64_ss(d, ah + 2 * ks, hs + 2 * ks, ks > 0);
        mma_m64n64_ss(d, al + 2 * ks, hs + 2 * ks, 1);
      }
      mma_commit();
      mma_wait<0>();
      reg_fence(d);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int u = 16 * warp + g + 8 * i;
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int r = 8 * j + 2 * cq + c;
          red[u * kFtRows + r] = fmaxf((d[4 * j + 2 * i + c] + d[4 * (j + 4) + 2 * i + c]) + b2[i], 0.f) * wdeep[i];
        }
    }
    __syncthreads();
    {  // 32 rows x 4 partial sums of 16 units
      const int r = tid & 31, part = tid >> 5;
      float s = 0.f;
#pragma unroll
      for (int u = 0; u < 16; ++u) s += red[(part * 16 + u) * kFtRows + r];
      zp[part * kFtRows + r] = s;
    }
    __syncthreads();
    if (tid < kFtRows) {
      const int row = row0 + tid;
      if (row < b.B) {
        const int G = p.n_genres;
        const int mid = checked_id(__ldg(b.movie_id + row), p.n_movies, b.err_flag);
        const int uid = checked_id(__ldg(b.user_id + row), p.n_users, b.err_flag);
        int ig = __ldg(b.movie_genre + row * 3), ug = __ldg(b.user_genre + row * 5);
        if (ig >= G) ig = -1;
        if (ug >= G) ug = -1;
        // one-hot block order (sorted column names): movieGenre1 | movieId | userGenre1 | userId
        float z = 0.f;
        if (ig >= 0) z += __ldg(p.first + ig);
        z += __ldg(p.first + G + mid);
        if (ug >= 0) z += __ldg(p.first + G + p.n_movies + ug);
        z += __ldg(p.first + (size_t)(2 * G + p.n_movies) + uid);
#pragma unroll
        for (int d = 0; d < 4; ++d) z = fmaf(dots[tid * 4 + d], p.wdot[d], z);
        z += ((zp[tid] + zp[kFtRows + tid]) + (zp[2 * kFtRows + tid] + zp[3 * kFtRows + tid])) + p.bout;
        store_score(b, row, sigmoidf_acc(z));
        if (b.logits) b.logits[row] = z;
      }
    }
    // the K padding of X was overwritten by H1 (K = 64): restore zeros for the next super-group
    __syncthreads();
    for (int i = tid; i < 2 * kFtRows * 4; i += 128) {
      const int r = i >> 2, ch = 4 + (i & 3);
      *reinterpret_cast<uint4*>(sc + FS_X + sw128_offset(r, ch)) = make_uint4(0, 0, 0, 0);
    }
  }
  if (!weights_ready) mbar_wait(&wbar, 0);
}

static size_t deepfm_tc_smem() { return 1024 + FIMG_BYTES + FS_BYTES; }

cudaError_t launch_deepfm_tc(const DeepFmParams& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  const int n_sg = (b.B + kFtRows - 1) / kFtRows;
  const int cap = 2 * p.num_sms;                         // two CTAs fit per SM
  const int grid = n_sg < cap ? n_sg : cap;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(128);
  cfg.dynamicSmemBytes = deepfm_tc_smem();
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  ++g_launch_count;
  return cudaLaunchKernelEx(&cfg, deepfm_tc_kernel, p, b);
}

cudaError_t setup_deepfm_tc_attributes() {
  return cudaFuncSetAttribute(deepfm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)deepfm_tc_smem());
}

}  // namespace srs
