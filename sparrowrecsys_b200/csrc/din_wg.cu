// din_wg.cu - DIN forward with the activation unit on Hopper warpgroup MMAs (wgmma), E padded
// to 32 or 64, any history length (64-position MMA tiles).
//
// Reference: TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DIN.py:125-167.  Same math as
// din.cu; what changes is where the per-(row, position) work of the activation unit runs:
//
//   * the movie table is stored pre-split, one row [EP x bf16 hi | EP x bf16 lo] per movie
//     (x = hi + lo, both round-to-nearest), so a gathered row IS an MMA operand row: history
//     rows go HBM/L2 -> shared memory by cp.async and are never touched by a CUDA core before
//     the MMA;
//   * activation unit: (h*c).Wp = h.(diag(c) Wp), so per batch row r the B operand
//         W_r = (Wsub + Wh) + diag(c_r) Wp            [32 units x EP]
//     is built once (fp32, then split to bf16 hi/lo) and 64 positions form one M = 64 tile:
//         D[64 x 32] = H_hi W_hi + H_lo W_hi + H_hi W_lo    (bf16x3, fp32 accumulate)
//   * gate (PReLU per position, Dense(1), sigmoid) on the accumulator registers, one quad of
//     lanes per position;
//   * pooling sum_t w_t h_t on a warpgroup MMA from the same shared-memory tile, read MN-major
//     (its 128-byte rows are positions): D[e'][n] = sum_t A[t][e'] Pb[n][t] with Pb's rows w hi and
//     w lo, so pooled = h_hi w_hi + h_lo w_hi + h_hi w_lo (bf16x3, as the activation unit);
//   * top MLP over the CTA's 32-row tile.  E <= 32: on wgmma, computed transposed like
//     embmlp_tc.cu - D[units x rows] = W^T X^T with W1^T (the 160 embedding columns of the tile) and
//     W2^T in shared memory as bf16 hi / lo images, the tile's hi and lo halves stacked along N, the
//     7 raw-scale numerics added in fp32 in the layer-1 epilogue, PReLU / Dense(1) / sigmoid on the
//     accumulator registers.  E <= 64: on CUDA cores (common.cuh::dense_layer); its W1 image would be
//     ~160 KB, and at cfg 5's T = 200 the activation unit dominates the tile.
//
// CTA = G warpgroups (DinWgLayout::G: 5 at E <= 32, 3 at E <= 64), 32 batch rows; warpgroup q owns rows
// q, q + G, ... and double-buffers its history tiles (the next tile's cp.async runs under this tile's MMA
// and epilogue; the ids of the tile after it are already on their way from HBM).  The per-row chain is
// latency-bound, so more warpgroups shorten each warpgroup's walk (7 or 6 rows at G = 5) without
// lengthening the chain.  At E <= 32 the 112 KB MLP image is not resident beside the warpgroups' buffers:
// they share one region, the image at its bottom and the buffers at its top, and the image bytes under the
// buffers are copied again in each tile once its activation unit is done (28 KB of W2^T at G = 5, in
// flight under Dense(128)).  The shared tile helpers that map threads generically (tile_side_features,
// stage_weights) use every warpgroup; dense_layer and row_dot (E <= 64) map 256 threads, and only
// warpgroups 0 and 1 issue the top MLP's Dense(128).  Shared memory: ~227 KB (E <= 32) / ~218 KB
// (E <= 64): one CTA per SM.
#include "kernels.h"
#include "wgmma.cuh"

namespace srs {
using namespace wg;

// 1 / x to about 1 ulp (rcp.approx): the gate weight it forms is rounded to 16 significant bits (bf16 hi + lo)
// before it is used, so the correctly rounded reciprocal's Newton steps and slow path buy nothing
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

constexpr int kWgRows = 32;       // rows per CTA (top-MLP tile height, as din.cu)
constexpr int kWgPos = 64;        // history positions per MMA tile
// warpgroups per CTA at E <= 32 (DESIGN §6 has the measurements that chose 5; a build with
// -DSRS_DIN_WG_GROUPS32=N measures another count)
#ifndef SRS_DIN_WG_GROUPS32
#define SRS_DIN_WG_GROUPS32 5
#endif

template <int EP>
struct DinWgLayout {
  static constexpr bool TC_MLP = EP == 32;                    // top MLP on wgmma
  // warpgroups per CTA: warpgroup q walks rows q, q + G, ... of the tile
  static constexpr int G = TC_MLP ? SRS_DIN_WG_GROUPS32 : 3;
  static constexpr int THREADS = 128 * G;
  static constexpr int KB = EP / 32;                          // 128-byte K blocks of a [hi | lo] row
  static constexpr uint32_t A_BYTES = KB * kWgPos * 128;      // one history tile
  static constexpr uint32_t B_BYTES = KB * 32 * 128;          // W_r, 32 unit rows
  static constexpr uint32_t WG_BYTES = 2 * A_BYTES + B_BYTES; // per warpgroup
  static constexpr uint32_t AU_BYTES = G * WG_BYTES;
  // top-MLP operand images (TC_MLP, written by model.cu::build_din_wg): W1^T [128 units][160 k] as k 0..127
  // in 2 K blocks, a hi and a lo image, then one tail K block whose 128-byte rows are [hi k 128..159 |
  // lo k 128..159]; W2^T [64 units][128 k] in 2 K blocks, a hi and a lo image
  static constexpr uint32_t IMG_W1_HI = 0, IMG_W1_LO = 32768, IMG_W1_TAIL = 65536;
  static constexpr uint32_t IMG_W2_HI = 81920, IMG_W2_LO = 98304;
  static constexpr uint32_t IMG_BYTES = TC_MLP ? 114688 : 0;
  static_assert(!TC_MLP || (IMG_W1_TAIL == 2 * 16384 * 2 && IMG_W2_HI == IMG_W1_TAIL + 16384 &&
                            IMG_BYTES == IMG_W2_LO + 2 * 8192), "top-MLP image layout");
  // X operand [32 rows hi | 32 rows lo][160 k] (3 K blocks), then the H1 operand [.. ][128 k] (2 K blocks)
  static constexpr uint32_t OP_KB_BYTES = 2 * kWgRows * 128;
  static constexpr int KP = 5 * EP + kNumPad, LDX = KP + 4, LDH1 = 128 + 4, LDH2 = 64 + 4;
  // fp32 region behind the operand tiles and images
  static constexpr int F_X = 0;
  static constexpr int F_H1 = F_X + kWgRows * LDX;                       // CUDA-core MLP only
  static constexpr int F_H2 = F_H1 + (TC_MLP ? 0 : kWgRows * LDH1);
  static constexpr int F_WH = F_H2 + (TC_MLP ? 0 : kWgRows * LDH2);    // [EP][32] Wsub + Wh
  static constexpr int F_WP = F_WH + EP * 32;                 // [EP][32] Wp
  static constexpr int F_WC = F_WP + EP * 32;                 // [EP][32] Wc - Wsub
  static constexpr int F_CST = F_WC + EP * 32;                // [32 rows][32 units] activation-unit constants
  static constexpr int F_WG = F_CST + kWgRows * 32;           // per warpgroup: pooled lo sums (EP = 32)
  static constexpr int F_WG_STRIDE = 32;
  static constexpr int F_RED = F_WG + G * F_WG_STRIDE;        // [4 warps][32 rows] Dense(1) partial sums
  static constexpr int F_END = F_RED + 4 * kWgRows;
  static constexpr uint32_t FS_BYTES = (uint32_t)F_END * sizeof(float);
  // pooling B operand per warpgroup, K-major [8 rows][64 positions] bf16: row 0 w hi, row 1 w lo, rows 2-7 zero.
  // They sit between the byte region and the fp32 region, where neither the image nor the X / H1 operand
  // reaches, so their zero rows are written once per CTA.
  static constexpr uint32_t PB_BYTES = 1024;
  // Byte region at the aligned base, in front of the pooling operands and the fp32 region.  E <= 64: the
  // warpgroups' history tiles and W_r.  E <= 32: every byte that one CTA per SM leaves (kSmemStatic: the static
  // mbarriers), the image at its bottom and the warpgroups' buffers at its top, the X / H1 operand over the last
  // of those.  The image bytes under the buffers (IMG_RELOAD) are copied again in every tile once its
  // activation unit is done; the rest (IMG_RESIDENT) is copied once per CTA.
  static constexpr uint32_t kSmemStatic = 64;
  static constexpr uint32_t REGION =
      TC_MLP ? (227u * 1024 - 1024 - kSmemStatic - G * PB_BYTES - FS_BYTES) / 1024 * 1024 : AU_BYTES;
  static constexpr uint32_t PB_OFF = REGION;                    // warpgroup q's pooling operand at PB_OFF + q PB_BYTES
  static constexpr uint32_t FS_OFF = PB_OFF + G * PB_BYTES;
  static constexpr uint32_t AU_OFF = REGION - AU_BYTES;         // warpgroup q's buffers at AU_OFF + q WG_BYTES
  static constexpr uint32_t OPS_OFF = REGION - 3 * OP_KB_BYTES; // X / H1 operand
  static constexpr uint32_t IMG_RESIDENT = AU_OFF < IMG_BYTES ? AU_OFF : IMG_BYTES;
  static constexpr uint32_t IMG_RELOAD = IMG_BYTES - IMG_RESIDENT;
  static constexpr bool RELOAD_IN_W2 = IMG_RESIDENT >= IMG_W2_HI;  // Dense(128) never waits for the reload
  static_assert(REGION >= AU_BYTES && AU_OFF % 1024 == 0 && IMG_RESIDENT % 16 == 0, "buffer alignment");
  static_assert(!TC_MLP || OPS_OFF >= IMG_BYTES, "the X / H1 operand must not overlap the image");
  static constexpr size_t SMEM = 1024 + FS_OFF + FS_BYTES;
  static_assert(SMEM + kSmemStatic <= 227 * 1024, "one CTA per SM must fit");
};

// byte offset of K byte `kb` (hi part: 2 e, lo part: 2 (EP + e)) of operand row `row` in a tile of
// `rows` rows: K blocks are `rows * 128` bytes apart
__device__ __forceinline__ uint32_t wg_kbyte(uint32_t row, uint32_t kb, uint32_t rows) {
  return (kb >> 7) * rows * 128u + sw128_offset(row, (kb & 127u) >> 4) + (kb & 15u);
}

// Top MLP of a 32-row tile on wgmma (E <= 32).  Xs holds the fp32 input tile; the X and H1 operands go
// over the history tiles at `ops`; `img` holds the W1^T / W2^T images: the resident part has landed once
// `res_bar` (if not null) completes, the reloaded part once `reload_bar` completes phase `parity`.  Ends
// with every score of the tile stored.
template <int EP>
__device__ __forceinline__ void top_mlp_wg(const DinParams& p, const BatchView& b, int row0, const float* Xs,
                                           uint8_t* ops, const uint8_t* img, float* red, uint64_t* res_bar,
                                           uint64_t* reload_bar, uint32_t parity, PhaseClock& clk) {
  using L = DinWgLayout<EP>;
  constexpr int KE = 5 * EP;                       // embedding columns of the tile: the MMAs' K
  static_assert(KE == 160, "W1 image: two full K blocks and a 32-wide tail");
  constexpr uint32_t KBB = L::OP_KB_BYTES, LO = kWgRows * 128;   // operand K block; lo rows follow the hi rows
  const int tid = threadIdx.x, q = tid >> 7, tw = tid & 127;
  const int warp = tw >> 5, lane = tw & 31, g = lane >> 2, cq = lane & 3;
  // X operand: tile columns 0 .. KE - 1 split to bf16 hi (operand rows 0..31) and lo (rows 32..63)
  for (int i = tid; i < kWgRows * KE / 2; i += L::THREADS) {
    const int r = i / (KE / 2), k = 2 * (i % (KE / 2));
    const float2 v = *reinterpret_cast<const float2*>(Xs + r * L::LDX + k);
    const Split2 s = split_pack(v.x, v.y);
    const uint32_t off = (uint32_t)(k >> 6) * KBB + sw128_offset(r, (k & 63) >> 3) + (k & 7) * 2;
    *reinterpret_cast<uint32_t*>(ops + off) = s.hi;
    *reinterpret_cast<uint32_t*>(ops + off + LO) = s.lo;
  }
  fence_async_smem();
  __syncthreads();
  clk.lap(PH_TOP_MLP);
  if (res_bar) mbar_wait(res_bar, 0);
  if (L::IMG_RELOAD > 0 && !L::RELOAD_IN_W2) mbar_wait(reload_bar, parity);
  clk.lap(PH_IMAGE_WAIT);
  const uint32_t s_img = smem_u32(img), s_op = smem_u32(ops);

  // ---- Dense(128) + PReLU: warpgroups 0 and 1, warpgroup q owns units 64 q .. 64 q + 63;
  // D[64 units x (32 rows hi | 32 rows lo)]
  {
    float d[32];
  #pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
    if (q < 2) {
      mma_fence();
    #pragma unroll
      for (int kb = 0; kb < 3; ++kb) {
        // k 0..127: hi and lo images; k 128..159: the tail block, hi at K byte 0 and lo at K byte 64 of its rows
        const uint64_t ah = kb < 2 ? desc_sw128(s_img + L::IMG_W1_HI + kb * 16384 + q * 8192)
                                   : desc_sw128(s_img + L::IMG_W1_TAIL + q * 8192);
        const uint64_t al = kb < 2 ? desc_sw128(s_img + L::IMG_W1_LO + kb * 16384 + q * 8192) : ah + 4;
        const uint64_t xs = desc_sw128(s_op + kb * KBB);
    #pragma unroll
        for (int ks = 0; ks < (kb < 2 ? 4 : 2); ++ks) {
          mma_m64n64_ss(d, ah + 2 * ks, xs + 2 * ks, kb > 0 || ks > 0);
          mma_m64n64_ss(d, al + 2 * ks, xs + 2 * ks, 1);
        }
      }
      mma_commit();
      mma_wait<0>();
      reg_fence(d);
    }
    __syncthreads();                               // both warpgroups' MMAs have read X: H1 goes over it
    // epilogue: units u = 64 q + 16 warp + g + 8 i, tile rows r = 8 j + 2 cq + c (hi: column r, lo: 32 + r)
  #pragma unroll
    for (int i = 0; i < 2 * (q < 2); ++i) {
      const int u = 64 * q + 16 * warp + g + 8 * i;
      const float bias = __ldg(p.b1 + u), slope = __ldg(p.a1 + u);
      float wn[kNumNumerics];
  #pragma unroll
      for (int n = 0; n < kNumNumerics; ++n) wn[n] = __ldg(p.W1 + (size_t)(KE + n) * 128 + u);
      const uint32_t koff = (uint32_t)(u >> 6) * KBB, chunk = (u & 63) >> 3, within = (u & 7) * 2;
  #pragma unroll
      for (int j = 0; j < 4; ++j)
  #pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int r = 8 * j + 2 * cq + c;
          const float* num = Xs + r * L::LDX + KE;
          float v = d[4 * j + 2 * i + c] + d[4 * (j + 4) + 2 * i + c] + bias;
  #pragma unroll
          for (int n = 0; n < kNumNumerics; ++n) v = fmaf(num[n], wn[n], v);
          v = v > 0.f ? v : slope * v;
          const __nv_bfloat16 vh = __float2bfloat16_rn(v);
          const uint32_t off = koff + sw128_offset(r, chunk) + within;
          *reinterpret_cast<__nv_bfloat16*>(ops + off) = vh;
          *reinterpret_cast<__nv_bfloat16*>(ops + off + LO) = __float2bfloat16_rn(v - __bfloat162float(vh));
        }
    }
    fence_async_smem();
    __syncthreads();
  }
  // ---- Dense(64) + PReLU, Dense(1), sigmoid: warpgroup 0, D[64 units x (32 rows hi | 32 rows lo)]
  if (q != 0) return;
  if (L::IMG_RELOAD > 0 && L::RELOAD_IN_W2) {      // the reloaded part is W2's: it flew under Dense(128)
    clk.lap(PH_TOP_MLP);
    mbar_wait(reload_bar, parity);
    clk.lap(PH_IMAGE_WAIT);
  }
  float d[32];
  #pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;
  float bias[2], slope[2], w3[2];                  // units u = 16 warp + g + 8 i, requested before the MMAs
  #pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int u = 16 * warp + g + 8 * i;
    bias[i] = __ldg(p.b2 + u);
    slope[i] = __ldg(p.a2 + u);
    w3[i] = __ldg(p.w3 + u);
  }
  mma_fence();
  #pragma unroll
  for (int kb = 0; kb < 2; ++kb) {
    const uint64_t ah = desc_sw128(s_img + L::IMG_W2_HI + kb * 8192);
    const uint64_t al = desc_sw128(s_img + L::IMG_W2_LO + kb * 8192);
    const uint64_t hs = desc_sw128(s_op + kb * KBB);
  #pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      mma_m64n64_ss(d, ah + 2 * ks, hs + 2 * ks, kb > 0 || ks > 0);
      mma_m64n64_ss(d, al + 2 * ks, hs + 2 * ks, 1);
    }
  }
  mma_commit();
  mma_wait<0>();
  reg_fence(d);
  float s[4][2];
  #pragma unroll
  for (int j = 0; j < 4; ++j) s[j][0] = s[j][1] = 0.f;
  #pragma unroll
  for (int i = 0; i < 2; ++i) {
  #pragma unroll
    for (int j = 0; j < 4; ++j)
  #pragma unroll
      for (int c = 0; c < 2; ++c) {
        float v = d[4 * j + 2 * i + c] + d[4 * (j + 4) + 2 * i + c] + bias[i];
        v = v > 0.f ? v : slope[i] * v;
        s[j][c] = fmaf(v, w3[i], s[j][c]);
      }
  }
  // sum over the 8 lanes of a column quad (g), then over the 4 warps in a fixed order
  #pragma unroll
  for (int j = 0; j < 4; ++j)
  #pragma unroll
    for (int c = 0; c < 2; ++c) {
      float v = s[j][c];
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (g == 0) red[warp * kWgRows + 8 * j + 2 * cq + c] = v;
    }
  named_sync(1, 128);
  if (tw < kWgRows) {
    const int row = row0 + tw;
    if (row < b.B) {
      const float z = ((red[tw] + red[kWgRows + tw]) + (red[2 * kWgRows + tw] + red[3 * kWgRows + tw])) + p.b3;
      store_score(b, row, sigmoidf_acc(z));
      if (b.logits) b.logits[row] = z;
    }
  }
}

template <int EP>
__global__ void __launch_bounds__(DinWgLayout<EP>::THREADS, 1) din_wg_kernel(DinParams p, BatchView b) {
  using L = DinWgLayout<EP>;
  constexpr int G = L::G, NT = L::THREADS;
  constexpr int KB = L::KB;
  constexpr int KS = EP / 16;                     // K steps per part (hi or lo)
  constexpr int CP = 8 * KB;                      // 16-byte chunks per split row
  constexpr int NCOPY = kWgPos * CP / 128;        // cp.async per thread per tile
  constexpr int OFF_UG = 0, OFF_U = EP, OFF_POOL = 2 * EP, OFF_C = 3 * EP, OFF_MG = 4 * EP, OFF_NUM = 5 * EP;
  extern __shared__ uint8_t raw[];
  __shared__ uint64_t res_bar, reload_bar;        // top-MLP image (TC_MLP): resident part / this tile's reload landed
  uint8_t* base = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
  uint8_t* img = base;
  float* fs = reinterpret_cast<float*>(base + L::FS_OFF);
  float* Xs = fs + L::F_X;
  float* H1 = fs + L::F_H1;
  float* H2 = fs + L::F_H2;
  const float* wh = fs + L::F_WH;
  const float* wp = fs + L::F_WP;
  const float* wc = fs + L::F_WC;
  float* cst_all = fs + L::F_CST;
  const int tid = threadIdx.x;
  const int q = tid >> 7, tw = tid & 127;
  const int warp = tw >> 5, lane = tw & 31, g = lane >> 2, cq = lane & 3;
  const int T = p.T, nch = (T + kWgPos - 1) / kWgPos;
  uint8_t* tiles = base + L::AU_OFF + q * L::WG_BYTES;   // history tiles 0, 1 | W_r
  uint8_t* Bt = tiles + 2 * L::A_BYTES;
  PhaseClock clk(tw == 0);
  // pooling B operand: w hi | w lo | 6 zero rows (128 threads x 8 B: the whole operand)
  reinterpret_cast<uint2*>(base + L::PB_OFF + q * L::PB_BYTES)[tw] = make_uint2(0u, 0u);

  bool weights_ready = !L::TC_MLP;
  uint32_t reload_parity = 0;
  if constexpr (L::TC_MLP) {
    if (tid == 0) {                               // visible to the waiters through the tile loop's first barrier
      mbar_init(&res_bar, 1);
      mbar_init(&reload_bar, 1);
      fence_mbar_init();
      mbar_arrive_expect_tx(&res_bar, L::IMG_RESIDENT);
      for (uint32_t off = 0; off < L::IMG_RESIDENT; off += 32768u)
        bulk_g2s(img + off, p.mlp_image + off, min(32768u, L::IMG_RESIDENT - off), &res_bar);
    }
  }
  stage_weights<NT>(fs + L::F_WH, p.au_wh, EP * 32);
  stage_weights<NT>(fs + L::F_WP, p.au_wp, EP * 32);
  stage_weights<NT>(fs + L::F_WC, p.au_wc, EP * 32);
  // persistent over the batch's 32-row tiles: one tile per CTA unless srs_model_set_sm_limit caps the grid
  const int n_tiles = (b.B + kWgRows - 1) / kWgRows;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int row0 = tile * kWgRows;
    // Warp 0 brings the lines of the tile's ids into L1 at once: the steps below that each wait for ids (side
    // features -> their rows, candidate id -> its row, history ids -> the first gathers) then find them there
    // instead of making their own HBM round trips one after the other.
    if (tid < kWgRows && row0 + tid < b.B) {
      const int row = row0 + tid, n = min(T, kWgPos);
      const int32_t* h = b.hist + (size_t)row * b.hist_stride;
      prefetch_l1(b.user_id + row);
      prefetch_l1(b.user_genre + row * 5);
      prefetch_l1(b.movie_genre + row * 3);
      prefetch_l1(b.movie_id + row);
      prefetch_l1(b.numerics + row * kNumNumerics);
      prefetch_l1(h);                                        // the first chunk's ids: at most 3 lines
      prefetch_l1(h + (n - 1) / 2);
      prefetch_l1(h + n - 1);
    }
    tile_side_features<EP, kWgRows, NT>(Xs, L::LDX, row0, b, p.user, p.ugenre, p.mgenre, p.n_users, p.n_genres,
                                        OFF_UG, OFF_U, OFF_MG, OFF_NUM);
    // candidate rows of the tile (ids pass through float32, DIN.py:95,125); rows past the batch end are zero
    for (int i = tid; i < kWgRows * EP / 4; i += NT) {
      const int r = i / (EP / 4), c4 = i % (EP / 4), row = row0 + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < b.B) {
        const int cid = checked_id(__float2int_rz(__int2float_rn(__ldg(b.movie_id + row))), p.n_movies, b.err_flag);
        v = ldg4(p.movie + (size_t)cid * EP + 4 * c4);
      } else {
        *reinterpret_cast<float4*>(Xs + r * L::LDX + OFF_POOL + 4 * c4) = v;
      }
      *reinterpret_cast<float4*>(Xs + r * L::LDX + OFF_C + 4 * c4) = v;
    }
    stage_wait();
    __syncthreads();
    // activation-unit constant of every row: cst[r][j] = au_b[j] + sum_e c_r[e] (Wc - Wsub)[e][j]
    for (int i = tid; i < kWgRows * 32; i += NT) {
      const int r = i >> 5, j = i & 31;
      const float* cv = Xs + r * L::LDX + OFF_C;
      float acc = __ldg(p.au_b + j);
  #pragma unroll 8
      for (int e = 0; e < EP; ++e) acc = fmaf(cv[e], wc[e * 32 + j], acc);
      cst_all[i] = acc;
    }
    __syncthreads();
    clk.lap(PH_TILE_INPUTS);
    // rows of this warpgroup: q, q + G, ...; the valid ones are a prefix
    int nrows = 0;
    for (int r = q; r < kWgRows; r += G)
      if (row0 + r < b.B) ++nrows;

    // gate constants of this thread's 8 accumulator columns 8 j + 2 cq + c
    float wout[8];
  #pragma unroll
    for (int j = 0; j < 4; ++j)
  #pragma unroll
      for (int c = 0; c < 2; ++c) wout[2 * j + c] = __ldg(p.au_wout + 8 * j + 2 * cq + c);

    const int n_items = nrows * nch;                // (row, 64-position chunk) pairs, chunk fastest
    // The history ids of an item are requested (into registers) two items before its rows are gathered,
    // so the HBM latency of the ids is not on the item chain.  Whether a slot is live is decided from its
    // position, never from the id value: every live id goes through the range check.
    // item k is chunk k % nch of the warpgroup's row k / nch; with one chunk per row (T <= 64) no division
    auto item_row = [&](int k) { return nch == 1 ? k : k / nch; };
    auto item_ch = [&](int k) { return nch == 1 ? 0 : k % nch; };
    auto item_nt = [&](int k) { return k < n_items ? min(kWgPos, T - item_ch(k) * kWgPos) : 0; };
    auto load_ids = [&](int k, int (&ids)[NCOPY]) {
      const int row = row0 + q + G * item_row(k), t0 = item_ch(k) * kWgPos, nt = item_nt(k);
      const int32_t* hrow = b.hist + (size_t)row * b.hist_stride + t0;
  #pragma unroll
      for (int n = 0; n < NCOPY; ++n) {
        const int pos = (tw + 128 * n) / CP;
        ids[n] = pos < nt ? __ldg(hrow + pos) : 0;
      }
    };
    // Every position of the tile is written: positions past nt are zero-filled, because the pooling MMA
    // reads them (with w = 0, which a stale NaN would still turn into NaN).  An out-of-range id is read as
    // row 0 and latches the error word, once per warp and item.
    auto gather = [&](int k, const int (&ids)[NCOPY]) {
      if (k >= n_items) return;
      uint8_t* A = tiles + (k & 1) * L::A_BYTES;
      const int nt = item_nt(k);
      bool bad = false;
  #pragma unroll
      for (int n = 0; n < NCOPY; ++n) {
        const int i = tw + 128 * n, pos = i / CP, c = i % CP;
        const int id = __float2int_rz(__int2float_rn(ids[n]));
        const bool in_range = static_cast<unsigned>(id) < static_cast<unsigned>(p.n_movies);
        bad |= !in_range;                                     // ids past nt are 0: never out of range
        cp_async16_zfill(A + (c >> 3) * (kWgPos * 128) + sw128_offset(pos, c & 7),
                         p.movie_split + (size_t)(in_range ? id : 0) * (CP * 16) + c * 16, pos < nt ? 16u : 0u);
      }
      if (__any_sync(0xffffffffu, bad) && lane == 0 && b.err_flag) atomicExch(b.err_flag, 1);
    };

    int ids_next[NCOPY];
    {
      int ids0[NCOPY];
      load_ids(0, ids0);
      load_ids(1, ids_next);
      gather(0, ids0);
    }
    cp_async_commit();
    const uint32_t pb_s = smem_u32(base + L::PB_OFF + q * L::PB_BYTES);
    float* pool_lo = fs + L::F_WG + q * L::F_WG_STRIDE;
    // W_r destinations of this thread (unit j = lane, element pair e = 2 warp + 8 n, K byte 4 warp + 16 n), the
    // same in every row: chunk n of row `lane`, byte 4 warp within it; its sources wh / wp [e][j]
    const uint32_t wr_row = smem_u32(Bt) + lane * 128u + 4u * warp, wr_sw = lane & 7u;
    const int wr_src = 2 * warp * 32 + lane;
    float slope[2][8], cstv[8];
    // pooled sums of the row so far: D[e'][n] = sum_t A[t][e'] Pb[n][t] for the operand columns e' of K block kb
    // (EP = 32: hi e | lo e; EP = 64: block 0 hi, block 1 lo) and n = w hi, w lo, added chunk by chunk
    float pacc[KB][4];
    for (int k = 0; k < n_items; ++k) {
      const int r = q + G * item_row(k), ch = item_ch(k), t0 = ch * kWgPos;
      const int nt = min(kWgPos, T - t0);
      float* xrow = Xs + r * L::LDX;
      const float* cst = cst_all + r * 32;
      if (ch == 0) {
        // B operand of the row: W_r = (Wsub + Wh) + diag(c_r) Wp, split to bf16 hi / lo.  Thread (warp, lane)
        // writes unit j = lane, element pairs e = 2 warp + 8 n: the lanes of a warp read 32 consecutive banks
        const float* cv = xrow + OFF_C + 2 * warp;
  #pragma unroll
        for (int n = 0; n < EP / 8; ++n) {
          const float2 c2 = *reinterpret_cast<const float2*>(cv + 8 * n);
          const float v0 = fmaf(c2.x, wp[wr_src + 256 * n], wh[wr_src + 256 * n]);
          const float v1 = fmaf(c2.y, wp[wr_src + 256 * n + 32], wh[wr_src + 256 * n + 32]);
          const Split2 s = split_pack(v0, v1);
          // the lo half of K byte kb sits at K byte 2 EP + kb: 64 bytes on in the same row (EP = 32, the
          // chunk index gains bit 2), or the next K block (EP = 64)
          const uint32_t dst = wr_row + ((n ^ wr_sw) << 4);
          st_shared_u32(dst, s.hi);
          st_shared_u32(EP == 32 ? dst ^ 64u : dst + 32u * 128u, s.lo);
        }
  #pragma unroll
        for (int j = 0; j < 4; ++j)
  #pragma unroll
          for (int c = 0; c < 2; ++c) cstv[2 * j + c] = cst[8 * j + 2 * cq + c];
        clk.lap(PH_W_BUILD);
      }
      gather(k + 1, ids_next);                                // its buffer's last reader finished before the
      cp_async_commit();                                      // closing barrier of item k - 1
      load_ids(k + 2, ids_next);
      // PReLU slopes of this thread's positions pr = 16 warp + g + 8 i and columns 8 j + 2 cq + c, times the
      // Dense(1) weights (the gate adds z wout or z slope wout), requested before the waits below; with one chunk
      // per row (T <= 64) they are the same for every row
      if (nch > 1 || k == 0) {
  #pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float* alpha = p.au_alpha + (size_t)min(t0 + 16 * warp + g + 8 * i, T - 1) * 32;
  #pragma unroll
          for (int j = 0; j < 4; ++j)
  #pragma unroll
            for (int c = 0; c < 2; ++c) slope[i][2 * j + c] = __ldg(alpha + 8 * j + 2 * cq + c) * wout[2 * j + c];
        }
      }
      clk.lap(PH_GATHER_ISSUE);
      cp_async_wait<1>();
      fence_async_smem();
      named_sync(1 + q, 128);                                 // tile k and W_r in place
      clk.lap(PH_GATHER_WAIT);

      // ---- activation unit: D[64 positions x 32 units], bf16x3
      float d[16];
  #pragma unroll
      for (int i = 0; i < 16; ++i) d[i] = 0.f;
      {
        const uint32_t sa = smem_u32(tiles + (k & 1) * L::A_BYTES), sb = smem_u32(Bt);
        mma_fence();
  #pragma unroll
        for (int s = 0; s < KS; ++s) {
          const uint32_t kh = 32 * s, kl = 2 * EP + 32 * s;   // K byte of the hi / lo step
          const uint64_t ah = desc_sw128(sa + (kh >> 7) * (kWgPos * 128) + (kh & 127));
          const uint64_t al = desc_sw128(sa + (kl >> 7) * (kWgPos * 128) + (kl & 127));
          const uint64_t bh = desc_sw128(sb + (kh >> 7) * (32 * 128) + (kh & 127));
          const uint64_t bl = desc_sw128(sb + (kl >> 7) * (32 * 128) + (kl & 127));
          mma_m64n32_ss(d, ah, bh, s > 0);
          mma_m64n32_ss(d, al, bh, 1);
          mma_m64n32_ss(d, ah, bl, 1);
        }
        mma_commit();
        mma_wait<0>();
        reg_fence(d);
      }
      clk.lap(PH_AU_MMA);
      // ---- gate: positions pr = 16 warp + g + 8 i; the quad of lanes sharing a position sums its 32 units
  #pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int pr = 16 * warp + g + 8 * i;
        float s = 0.f;
  #pragma unroll
        for (int j = 0; j < 4; ++j)
  #pragma unroll
          for (int c = 0; c < 2; ++c) {
            const float z = d[4 * j + 2 * i + c] + cstv[2 * j + c];
            s = fmaf(z, z > 0.f ? wout[2 * j + c] : slope[i][2 * j + c], s);
          }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        // w split to bf16 hi / lo into rows 0 and 1 of the pooling operand (K byte 2 pr); w = 0 past nt
        const float w = pr < nt ? rcp_approx(1.f + __expf(-(s + p.au_bout))) : 0.f;
        if (cq == 0) {
          const __nv_bfloat16 wh16 = __float2bfloat16_rn(w);
          const __nv_bfloat16 wl16 = __float2bfloat16_rn(w - __bfloat162float(wh16));
          st_shared_u16(pb_s + sw128_offset(0, pr >> 3) + 2 * (pr & 7), __bfloat16_as_ushort(wh16));
          st_shared_u16(pb_s + sw128_offset(1, pr >> 3) + 2 * (pr & 7), __bfloat16_as_ushort(wl16));
        }
      }
      fence_async_smem();
      named_sync(1 + q, 128);                                 // w in place
      clk.lap(PH_GATE);
      // ---- pooling: D (+)= A^T Pb over the tile's 64 positions, A read MN-major (its 128-byte rows are
      // positions); products h_hi w_hi, h_lo w_hi, h_hi w_lo as in the activation unit
      {
        // (an accumulator set that stayed live across the next activation-unit MMAs would make ptxas spill)
        const uint32_t sa = smem_u32(tiles + (k & 1) * L::A_BYTES), sp = pb_s;
        float pd[KB][4];
        mma_fence();
  #pragma unroll
        for (int s = 0; s < kWgPos / 16; ++s)
  #pragma unroll
          for (int kb = 0; kb < KB; ++kb)
            mma_m64n8_ss_amn(pd[kb], desc_sw128_mn(sa + kb * (kWgPos * 128) + s * 2048), desc_sw128(sp + 32 * s),
                             s > 0);
        mma_commit();
        mma_wait<0>();
  #pragma unroll
        for (int kb = 0; kb < KB; ++kb) {
          reg_fence(pd[kb]);
  #pragma unroll
          for (int i = 0; i < 4; ++i) pacc[kb][i] = ch > 0 ? pacc[kb][i] + pd[kb][i] : pd[kb][i];
        }
      }
      // lanes cq = 0 hold columns w hi (pacc[.][0], [2]) and w lo ([1], [3]) of operand columns 16 warp + g (+ 8);
      // at EP = 32 the lo elements' sums (columns 32 + e) are in warps 2 and 3 and go through shared memory
      const bool last = ch == nch - 1;
      if (EP == 32 && last && warp >= 2 && cq == 0) {
        pool_lo[16 * (warp - 2) + g] = pacc[0][0];
        pool_lo[16 * (warp - 2) + g + 8] = pacc[0][2];
      }
      named_sync(1 + q, 128);                                 // tile k, Pb and W_r free again
      if (last && cq == 0 && (EP == 64 || warp < 2)) {
  #pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int e = 16 * warp + g + 8 * i;
          const float lo_whi = EP == 32 ? pool_lo[e] : pacc[KB - 1][2 * i];
          xrow[OFF_POOL + e] = (pacc[0][2 * i] + lo_whi) + pacc[0][2 * i + 1];
        }
      }
      clk.lap(PH_POOL);
    }
    if constexpr (L::TC_MLP) {
      // the top MLP's epilogue constants (b1, a1, the numerics' rows of W1, b2, a2, w3: 42 lines) come into L1
      // while the warpgroups wait for the one with the most rows
      if (tw < 42) {
        const float* src = tw < 4 ? p.b1 + 32 * tw : tw < 8 ? p.a1 + 32 * (tw - 4)
                         : tw < 36 ? p.W1 + (size_t)(5 * EP + (tw - 8) / 4) * 128 + 32 * ((tw - 8) % 4)
                         : tw < 38 ? p.b2 + 32 * (tw - 36) : tw < 40 ? p.a2 + 32 * (tw - 38) : p.w3 + 32 * (tw - 40);
        prefetch_l1(src);
      }
    }
    cp_async_wait<0>();
    __syncthreads();
    clk.lap(PH_ROW_IMBALANCE);

    // ---- top MLP on the tile ----------------------------------------------------------
    if constexpr (L::TC_MLP) {
      if (L::IMG_RELOAD > 0 && tid == 0) {
        // every warpgroup is past its last wgmma and shared-memory access of the history tiles (the barrier
        // above); the fence orders those before the bulk copy that writes the image's top over them
        fence_async_smem();
        mbar_arrive_expect_tx(&reload_bar, L::IMG_RELOAD);
        for (uint32_t off = L::IMG_RESIDENT; off < L::IMG_BYTES; off += 32768u)
          bulk_g2s(img + off, p.mlp_image + off, min(32768u, L::IMG_BYTES - off), &reload_bar);
      }
      top_mlp_wg<EP>(p, b, row0, Xs, base + L::OPS_OFF, img, fs + L::F_RED, weights_ready ? nullptr : &res_bar,
                     &reload_bar, reload_parity, clk);
      weights_ready = true;
      reload_parity ^= 1u;
    } else {
      if (tid < kThreads) dense_layer<kWgRows, 128, 2, 8>(Xs, L::LDX, L::KP, p.W1, p.b1, ACT_PRELU, p.a1, H1, L::LDH1);
      __syncthreads();
      if (tid < kThreads) dense_layer<kWgRows, 64, 1, 8>(H1, L::LDH1, 128, p.W2, p.b2, ACT_PRELU, p.a2, H2, L::LDH2);
      __syncthreads();
      if (tid < kThreads) row_dot<kWgRows>(H2, L::LDH2, 64, p.w3, [&](int r, float s) {
        const int row = row0 + r;
        if (row >= b.B) return;
        const float z = s + p.b3;
        store_score(b, row, sigmoidf_acc(z));
        if (b.logits) b.logits[row] = z;
      });
    }
    __syncthreads();                              // the next tile reuses every buffer
    clk.lap(PH_TOP_MLP);
  }
  // no bulk copy may outlive the CTA: each tile waited for its reload, and the first for the resident part
  // (the grid never exceeds the tile count, so every CTA has a tile)
  gather_signal_tail(b);                          // spanning ranking call: publish "slice complete"
}

// fp32 table [rows][EP] -> [rows][EP x bf16 hi | EP x bf16 lo]
template <int EP>
__global__ void split_table_kernel(const float* __restrict__ src, uint32_t* __restrict__ dst, int64_t n_pairs) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // pair index: row * EP / 2 + pair
  if (i >= n_pairs) return;
  const int64_t row = i / (EP / 2);
  const int pr = (int)(i % (EP / 2));
  const float2 v = *reinterpret_cast<const float2*>(src + row * EP + 2 * pr);
  const Split2 s = split_pack(v.x, v.y);
  dst[row * EP + pr] = s.hi;
  dst[row * EP + EP / 2 + pr] = s.lo;
}

cudaError_t launch_split_table(const float* src, void* dst, int64_t rows, int EP, cudaStream_t s) {
  const int64_t n_pairs = rows * (EP / 2);
  const int threads = 256;
  const int64_t blocks = (n_pairs + threads - 1) / threads;
  if (EP == 32) split_table_kernel<32><<<(unsigned)blocks, threads, 0, s>>>(src, reinterpret_cast<uint32_t*>(dst), n_pairs);
  else if (EP == 64) split_table_kernel<64><<<(unsigned)blocks, threads, 0, s>>>(src, reinterpret_cast<uint32_t*>(dst), n_pairs);
  else return cudaErrorInvalidValue;
  ++g_launch_count;
  return cudaGetLastError();
}

cudaError_t launch_din_wg(const DinParams& p, const BatchView& b, cudaStream_t s) {
  if (b.B <= 0) return cudaSuccess;
  const int n_tiles = (b.B + kWgRows - 1) / kWgRows;
  const int blocks = p.max_ctas > 0 && p.max_ctas < n_tiles ? p.max_ctas : n_tiles;
  ++g_launch_count;
  if (p.EP == 32) din_wg_kernel<32><<<blocks, DinWgLayout<32>::THREADS, DinWgLayout<32>::SMEM, s>>>(p, b);
  else if (p.EP == 64) din_wg_kernel<64><<<blocks, DinWgLayout<64>::THREADS, DinWgLayout<64>::SMEM, s>>>(p, b);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

#ifdef SRS_DIN_PHASES
cudaError_t din_wg_take_phases(unsigned long long* out) { return din_phases_take(out); }
#endif

cudaError_t setup_din_wg_attributes() {
  cudaError_t e = cudaFuncSetAttribute(din_wg_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)DinWgLayout<32>::SMEM);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(din_wg_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)DinWgLayout<64>::SMEM);
}

}  // namespace srs
