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
// CTA = G warpgroups (DinWgLayout::G: 4 at E <= 32, 3 at E <= 64), 32 batch rows; warpgroup q owns rows
// q, q + G, ... and walks them in items of R rows at one 64-position chunk (DinWgLayout::R: 2 at E <= 32, 1 at
// E <= 64), double-buffering the items' history tiles.  The rows of a pair share its barriers, its gather wait
// and its two MMA round trips (both rows' MMAs in one commit group, waited with wait_group 0).  The work that
// does not depend on those MMAs runs while they are in flight: the next item's gathers (and the ids of the item
// after it) are issued under the activation-unit MMAs, the next row's W_r is built under the pooling MMAs.
// At E <= 32 the 112 KB MLP image is not resident beside the warpgroups' buffers: they share one region, the
// image at its bottom and the buffers at its top, and the image bytes under the buffers (94 KB at G = 4,
// R = 2) are copied again in each tile once its activation unit is done, W1^T's
// part (if any) first on its own barrier so that W2^T's flies under Dense(128).  At E <= 32 a tile's inputs wait
// on no CTA-wide barrier (after the CTA's first tile): each warpgroup copies the candidate rows of its own rows
// and computes their activation-unit constants, and the side features, which only the top MLP reads, are copied
// by cp.async that the walk's gather waits cover.  At E <= 64 the CTA copies them all between two barriers.
// The shared tile helpers that map threads generically (tile_side_features, stage_weights) use every
// warpgroup; dense_layer and row_dot (E <= 64) map 256 threads, and only warpgroups 0 and 1 issue the top
// MLP's Dense(128).  Shared memory: ~227 KB (E <= 32) / ~218 KB
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
// warpgroups per CTA and batch rows per warpgroup item at E <= 32 (DESIGN §6 has the measurements that chose
// 4 and 2; a build with -DSRS_DIN_WG_GROUPS32=N or -DSRS_DIN_WG_ROWS32=N measures another count)
#ifndef SRS_DIN_WG_GROUPS32
#define SRS_DIN_WG_GROUPS32 4
#endif
#ifndef SRS_DIN_WG_ROWS32
#define SRS_DIN_WG_ROWS32 2
#endif

template <int EP>
struct DinWgLayout {
  static constexpr bool TC_MLP = EP == 32;                    // top MLP on wgmma
  // warpgroups per CTA: warpgroup q walks rows q, q + G, ... of the tile, R of them per item
  static constexpr int G = TC_MLP ? SRS_DIN_WG_GROUPS32 : 3;
  static constexpr int R = TC_MLP ? SRS_DIN_WG_ROWS32 : 1;
  static_assert(R >= 1 && R <= 2, "one or two rows per item");
  static constexpr int THREADS = 128 * G;
  static constexpr int KB = EP / 32;                          // 128-byte K blocks of a [hi | lo] row
  static constexpr uint32_t A_BYTES = KB * kWgPos * 128;      // one history tile
  static constexpr uint32_t B_BYTES = KB * 32 * 128;          // W_r, 32 unit rows
  // per warpgroup: two item buffers of R history tiles each, then R W_r operands
  static constexpr uint32_t WG_BYTES = 2 * R * A_BYTES + R * B_BYTES;
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
  static constexpr int F_WG = F_CST + kWgRows * 32;           // per warpgroup: pooled lo sums of R rows (EP = 32)
  static constexpr int F_WG_STRIDE = 32 * R;
  static constexpr int F_RED = F_WG + G * F_WG_STRIDE;        // [4 warps][32 rows] Dense(1) partial sums
  static constexpr int F_END = F_RED + 4 * kWgRows;
  static constexpr uint32_t FS_BYTES = (uint32_t)F_END * sizeof(float);
  // pooling B operand per item row, K-major [8 rows][64 positions] bf16: row 0 w hi, row 1 w lo, rows 2-7 zero.
  // They sit between the byte region and the fp32 region, where neither the image nor the X / H1 operand
  // reaches, so their zero rows are written once per CTA.
  static constexpr uint32_t PB_BYTES = 1024;
  static constexpr uint32_t PB_WG_BYTES = R * PB_BYTES;        // per warpgroup
  // Byte region at the aligned base, in front of the pooling operands and the fp32 region.  E <= 64: the
  // warpgroups' history tiles and W_r.  E <= 32: every byte that one CTA per SM leaves (kSmemStatic: the static
  // mbarriers), the image at its bottom and the warpgroups' buffers at its top, the X / H1 operand over the last
  // of those.  The image bytes under the buffers (IMG_RELOAD) are copied again in every tile once its
  // activation unit is done, W1^T's part (RELOAD_W1) first and on its own barrier, so that the copy of W2^T's
  // part (RELOAD_W2) still flies under Dense(128); the rest (IMG_RESIDENT) is copied once per CTA.
  static constexpr uint32_t kSmemStatic = 64;
  static constexpr uint32_t REGION =
      TC_MLP ? (227u * 1024 - 1024 - kSmemStatic - G * PB_WG_BYTES - FS_BYTES) / 1024 * 1024 : AU_BYTES;
  static constexpr uint32_t PB_OFF = REGION;                    // row s of warpgroup q: PB_OFF + q PB_WG_BYTES + s PB_BYTES
  static constexpr uint32_t FS_OFF = PB_OFF + G * PB_WG_BYTES;
  static constexpr uint32_t AU_OFF = REGION - AU_BYTES;         // warpgroup q's buffers at AU_OFF + q WG_BYTES
  static constexpr uint32_t OPS_OFF = REGION - 3 * OP_KB_BYTES; // X / H1 operand
  static constexpr uint32_t IMG_RESIDENT = AU_OFF < IMG_BYTES ? AU_OFF : IMG_BYTES;
  static constexpr uint32_t IMG_RELOAD = IMG_BYTES - IMG_RESIDENT;
  static constexpr uint32_t RELOAD_W1 = TC_MLP && IMG_RESIDENT < IMG_W2_HI ? IMG_W2_HI - IMG_RESIDENT : 0;
  static constexpr uint32_t RELOAD_W2_OFF = IMG_RESIDENT + RELOAD_W1;
  static constexpr uint32_t RELOAD_W2 = IMG_RELOAD - RELOAD_W1;
  static_assert(REGION >= AU_BYTES && AU_OFF % 1024 == 0 && IMG_RESIDENT % 16 == 0, "buffer alignment");
  static_assert(WG_BYTES % 1024 == 0 && (2 * R * A_BYTES) % 1024 == 0, "SW128 operands sit on 1 KB boundaries");
  static_assert(!TC_MLP || OPS_OFF >= IMG_BYTES, "the X / H1 operand must not overlap the image");
  static_assert(!TC_MLP || (RELOAD_W2_OFF >= IMG_W2_HI && RELOAD_W2_OFF + RELOAD_W2 == IMG_BYTES &&
                            RELOAD_W2_OFF % 16 == 0), "reload split at W2^T");
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
// `res_bar` (if not null) completes, the reloaded parts of W1^T and W2^T once `reload_bar[0]` and
// `reload_bar[1]` complete phase `parity`.  Ends with every score of the tile stored.
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
  if (L::RELOAD_W1 > 0) mbar_wait(&reload_bar[0], parity);
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
  if (L::RELOAD_W2 > 0) {                          // W2's reloaded part flew under Dense(128)
    clk.lap(PH_TOP_MLP);
    mbar_wait(&reload_bar[1], parity);
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
  constexpr int G = L::G, R = L::R, NT = L::THREADS;
  constexpr int KB = L::KB;
  constexpr int KS = EP / 16;                     // K steps per part (hi or lo)
  constexpr int CP = 8 * KB;                      // 16-byte chunks per split row
  constexpr int NCOPY = kWgPos * CP / 128;        // cp.async per thread per tile
  constexpr int NR = (kWgRows + G - 1) / G;       // most rows of a tile a warpgroup owns
  constexpr int OFF_UG = 0, OFF_U = EP, OFF_POOL = 2 * EP, OFF_C = 3 * EP, OFF_MG = 4 * EP, OFF_NUM = 5 * EP;
  extern __shared__ uint8_t raw[];
  // top-MLP image (TC_MLP): resident part / this tile's reload of W1^T's and of W2^T's part landed
  __shared__ uint64_t res_bar, reload_bar[2];
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
  // history tiles of item buffer 0 (rows 0 .. R - 1), of buffer 1 | W_r of rows 0 .. R - 1
  uint8_t* tiles = base + L::AU_OFF + q * L::WG_BYTES;
  uint8_t* Bt = tiles + 2 * R * L::A_BYTES;
  PhaseClock clk(tw == 0);
  // pooling B operands: w hi | w lo | 6 zero rows (128 threads x 8 B: one whole operand)
  #pragma unroll
  for (int s = 0; s < R; ++s)
    reinterpret_cast<uint2*>(base + L::PB_OFF + q * L::PB_WG_BYTES + s * L::PB_BYTES)[tw] = make_uint2(0u, 0u);

  bool weights_ready = !L::TC_MLP;
  uint32_t reload_parity = 0;
  if constexpr (L::TC_MLP) {
    if (tid == 0) {                               // visible to the waiters through the tile loop's first barrier
      mbar_init(&res_bar, 1);
      mbar_init(&reload_bar[0], 1);
      mbar_init(&reload_bar[1], 1);
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
    if constexpr (!L::TC_MLP) {
      // E <= 64: the tile's inputs by the whole CTA, between two CTA-wide barriers (DESIGN §4.1: the per-warpgroup
      // flow below measured 1 % slower at cfg 5, whose walk of 44 items per warpgroup dominates the tile)
      tile_side_features<EP, kWgRows, NT, true>(Xs, L::LDX, row0, b, p.user, p.ugenre, p.mgenre, p.n_users,
                                                p.n_genres, OFF_UG, OFF_U, OFF_MG, OFF_NUM);
      // candidate rows of the tile (ids pass through float32, DIN.py:95,125); rows past the batch end are zero
      for (int i = tid; i < kWgRows * EP / 4; i += NT) {
        const int r = i / (EP / 4), c4 = i % (EP / 4), row = row0 + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < b.B) {
          const int cid =
              checked_id(__float2int_rz(__int2float_rn(__ldg(b.movie_id + row))), p.n_movies, b.err_flag);
          v = ldg4(p.movie + (size_t)cid * EP + 4 * c4);
        } else {
          *reinterpret_cast<float4*>(Xs + r * L::LDX + OFF_POOL + 4 * c4) = v;
        }
        *reinterpret_cast<float4*>(Xs + r * L::LDX + OFF_C + 4 * c4) = v;
      }
      stage_wait();                               // the staged weights and the side features
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
    }
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

    // An item is a pair (R = 2) of the warpgroup's rows at one 64-position chunk, chunk fastest: item k is chunk
    // k % nch of rows q + G (R i + s), s < R, with i = k / nch.  Row s of the pair is live if R i + s < nrows; the
    // pair's first row always is.  A row that is not (the last pair of a warpgroup with an odd row count) has no
    // W_r build, gathers, gate or stores; nothing reads its buffers.  Its MMAs are still issued, on row 0's
    // operands, and their sums dropped: wgmmas skipped in a branch make ptxas serialise every wgmma (C7520).
    const int n_items = (nrows + R - 1) / R * nch;
    // The history ids of an item are requested (into registers) two items before its rows are gathered,
    // so the HBM latency of the ids is not on the item chain.  Whether a slot is live is decided from its
    // position, never from the id value: every live id goes through the range check.  The ids are read once
    // and take no L1 line (ldg_stream): L1 stays with the embedding rows the gathers read again (DESIGN §4.1).
    // With one chunk per row (T <= 64) the item is the pair: no division
    auto item_pair = [&](int k) { return nch == 1 ? k : k / nch; };
    auto item_ch = [&](int k) { return nch == 1 ? 0 : k % nch; };
    auto row_live = [&](int i, int s) { return s == 0 || R * i + s < nrows; };
    auto item_nt = [&](int k) { return k < n_items ? min(kWgPos, T - item_ch(k) * kWgPos) : 0; };
    auto load_ids = [&](int k, int (&ids)[R][NCOPY]) {
      const int i = item_pair(k), t0 = item_ch(k) * kWgPos, nt = item_nt(k);
  #pragma unroll
      for (int s = 0; s < R; ++s) {
        const int row = row0 + q + G * (R * i + s), nts = row_live(i, s) ? nt : 0;
        const int32_t* hrow = b.hist + (size_t)row * b.hist_stride + t0;
  #pragma unroll
        for (int n = 0; n < NCOPY; ++n) {
          const int pos = (tw + 128 * n) / CP;
          ids[s][n] = pos < nts ? ldg_stream(hrow + pos) : 0;
        }
      }
    };
    // Every position of a live row's tile is written: positions past nt are zero-filled, because the pooling MMA
    // reads them (with w = 0, which a stale NaN would still turn into NaN).  An out-of-range id is read as
    // row 0 and latches the error word, once per warp and item.
    auto gather = [&](int k, const int (&ids)[R][NCOPY]) {
      if (k >= n_items) return;
      uint8_t* A = tiles + (k & 1) * (R * L::A_BYTES);
      const int i = item_pair(k), nt = item_nt(k);
      bool bad = false;
  #pragma unroll
      for (int s = 0; s < R; ++s) {
        if (!row_live(i, s)) continue;
  #pragma unroll
        for (int n = 0; n < NCOPY; ++n) {
          const int t = tw + 128 * n, pos = t / CP, c = t % CP;
          const int id = __float2int_rz(__int2float_rn(ids[s][n]));
          const bool in_range = static_cast<unsigned>(id) < static_cast<unsigned>(p.n_movies);
          bad |= !in_range;                                   // ids past nt are 0: never out of range
          cp_async16_zfill(A + s * L::A_BYTES + (c >> 3) * (kWgPos * 128) + sw128_offset(pos, c & 7),
                           p.movie_split + (size_t)(in_range ? id : 0) * (CP * 16) + c * 16, pos < nt ? 16u : 0u);
        }
      }
      if (__any_sync(0xffffffffu, bad) && lane == 0 && b.err_flag) atomicExch(b.err_flag, 1);
    };

    // E <= 32: tile inputs per warpgroup.  Warpgroup q's walk reads the candidate rows and activation-unit
    // constants of its own rows only, so it copies and computes those alone and waits for itself; the side features
    // are read by the top MLP only, so their copies are issued with the first gathers and waited for by the walk's
    // first gather wait (or the wait before the top MLP).  The history ids are requested first, so that their round
    // trip overlaps the others.
    int ids_next[R][NCOPY];
    {
      int ids0[R][NCOPY];
      load_ids(0, ids0);
      load_ids(1, ids_next);
      if constexpr (L::TC_MLP) {
        // candidate rows (ids pass through float32, DIN.py:95,125); rows past the batch end are zero.  Their commit
        // group also holds the staged weights in the CTA's first tile.
        for (int i = tw; i < NR * (EP / 4); i += 128) {
          const int r = q + G * (i / (EP / 4)), c4 = i % (EP / 4), row = row0 + r;
          if (r >= kWgRows) break;
          const bool in = row < b.B;
          const int cid =
              in ? checked_id(__float2int_rz(__int2float_rn(__ldg(b.movie_id + row))), p.n_movies, b.err_flag) : 0;
          cp_async16_zfill(Xs + r * L::LDX + OFF_C + 4 * c4, p.movie + (size_t)cid * EP + 4 * c4, in ? 16u : 0u);
          if (!in)
            *reinterpret_cast<float4*>(Xs + r * L::LDX + OFF_POOL + 4 * c4) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        cp_async_commit();
        tile_side_features<EP, kWgRows, NT, true>(Xs, L::LDX, row0, b, p.user, p.ugenre, p.mgenre, p.n_users,
                                                  p.n_genres, OFF_UG, OFF_U, OFF_MG, OFF_NUM);
      }
      gather(0, ids0);
    }
    cp_async_commit();
    if constexpr (L::TC_MLP) {
      cp_async_wait<1>();                         // the candidate rows (and in the first tile the staged weights)
      // every warpgroup reads all of the staged weights: the CTA's first tile waits for the CTA, later ones for the
      // warpgroup
      if (tile == blockIdx.x) __syncthreads();
      else named_sync(1 + q, 128);
      // activation-unit constants of the warpgroup's rows: cst[r][j] = au_b[j] + sum_e c_r[e] (Wc - Wsub)[e][j]
      for (int i = tw; i < NR * 32; i += 128) {
        const int r = q + G * (i >> 5), j = i & 31;
        if (r >= kWgRows) break;
        const float* cv = Xs + r * L::LDX + OFF_C;
        float acc = __ldg(p.au_b + j);
  #pragma unroll 8
        for (int e = 0; e < EP; ++e) acc = fmaf(cv[e], wc[e * 32 + j], acc);
        cst_all[r * 32 + j] = acc;
      }
      named_sync(1 + q, 128);
      clk.lap(PH_TILE_INPUTS);
    }
    // per item row s: pooling operand at pb_s + s PB_BYTES, pooled lo sums at pool_lo + 32 s, W_r at + s B_BYTES
    const uint32_t pb_s = smem_u32(base + L::PB_OFF + q * L::PB_WG_BYTES);
    float* pool_lo = fs + L::F_WG + q * L::F_WG_STRIDE;
    // W_r destinations of this thread (unit j = lane, element pair e = 2 warp + 8 n, K byte 4 warp + 16 n), the
    // same in every row: chunk n of row `lane`, byte 4 warp within it; its sources wh / wp [e][j]
    const uint32_t wr_row = smem_u32(Bt) + lane * 128u + 4u * warp, wr_sw = lane & 7u;
    const int wr_src = 2 * warp * 32 + lane;
    float slope[2][8], cstv[R][8];
    // B operand of each live row of item k: W_r = (Wsub + Wh) + diag(c_r) Wp, split to bf16 hi / lo, and the row's
    // gate constants.  Thread (warp, lane) writes unit j = lane, element pairs e = 2 warp + 8 n: the lanes of a
    // warp read 32 consecutive banks
    auto build_wr = [&](int k) {
      const int i = item_pair(k);
  #pragma unroll
      for (int s = 0; s < R; ++s) {
        if (!row_live(i, s)) continue;
        const int r = q + G * (R * i + s);
        const float* cv = Xs + r * L::LDX + OFF_C + 2 * warp;
  #pragma unroll
        for (int n = 0; n < EP / 8; ++n) {
          const float2 c2 = *reinterpret_cast<const float2*>(cv + 8 * n);
          const float v0 = fmaf(c2.x, wp[wr_src + 256 * n], wh[wr_src + 256 * n]);
          const float v1 = fmaf(c2.y, wp[wr_src + 256 * n + 32], wh[wr_src + 256 * n + 32]);
          const Split2 sp = split_pack(v0, v1);
          // the lo half of K byte kb sits at K byte 2 EP + kb: 64 bytes on in the same row (EP = 32, the
          // chunk index gains bit 2), or the next K block (EP = 64)
          const uint32_t dst = wr_row + s * L::B_BYTES + ((n ^ wr_sw) << 4);
          st_shared_u32(dst, sp.hi);
          st_shared_u32(EP == 32 ? dst ^ 64u : dst + 32u * 128u, sp.lo);
        }
        const float* cst = cst_all + r * 32;
  #pragma unroll
        for (int j = 0; j < 4; ++j)
  #pragma unroll
          for (int c = 0; c < 2; ++c) cstv[s][2 * j + c] = cst[8 * j + 2 * cq + c];
      }
    };
    if (n_items > 0) build_wr(0);
    clk.lap(PH_W_BUILD);
    // pooled sums of each row so far: D[e'][n] = sum_t A[t][e'] Pb[n][t] for the operand columns e' of K block kb
    // (EP = 32: hi e | lo e; EP = 64: block 0 hi, block 1 lo) and n = w hi, w lo, added chunk by chunk
    float pacc[R][KB][4];
    for (int k = 0; k < n_items; ++k) {
      const int i = item_pair(k), ch = item_ch(k), t0 = ch * kWgPos;
      const int nt = min(kWgPos, T - t0);
      bool live[R];
      int r[R];
  #pragma unroll
      for (int s = 0; s < R; ++s) {
        live[s] = row_live(i, s);
        r[s] = q + G * (R * i + s);
      }
      // PReLU slopes of this thread's positions pr = 16 warp + g + 8 i and columns 8 j + 2 cq + c, times the
      // Dense(1) weights (the gate adds z wout or z slope wout), requested before the waits below; the same for
      // both rows of an item, and with one chunk per row (T <= 64) for every item
      if (nch > 1 || k == 0) {
  #pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float* alpha = p.au_alpha + (size_t)min(t0 + 16 * warp + g + 8 * h, T - 1) * 32;
  #pragma unroll
          for (int j = 0; j < 4; ++j)
  #pragma unroll
            for (int c = 0; c < 2; ++c) slope[h][2 * j + c] = __ldg(alpha + 8 * j + 2 * cq + c) * wout[2 * j + c];
        }
      }
      cp_async_wait<0>();
      fence_async_smem();
      named_sync(1 + q, 128);                                 // tiles of item k and W_r in place
      clk.lap(PH_GATHER_WAIT);

      const uint32_t sa = smem_u32(tiles + (k & 1) * (R * L::A_BYTES));
      // ---- activation unit: D[64 positions x 32 units] per row, bf16x3; the rows' MMAs in one commit group
      float d[R][16];
  #pragma unroll
      for (int s = 0; s < R; ++s)
  #pragma unroll
        for (int e = 0; e < 16; ++e) d[s][e] = 0.f;
      {
        mma_fence();
  #pragma unroll
        for (int s = 0; s < R; ++s) {
          // a row that is not live reads row 0's operands (so does its pooling below)
          const uint32_t sas = live[s] ? sa + s * L::A_BYTES : sa;
          const uint32_t sb = smem_u32(Bt) + (live[s] ? s * L::B_BYTES : 0u);
  #pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            const uint32_t kh = 32 * ks, kl = 2 * EP + 32 * ks;   // K byte of the hi / lo step
            const uint64_t ah = desc_sw128(sas + (kh >> 7) * (kWgPos * 128) + (kh & 127));
            const uint64_t al = desc_sw128(sas + (kl >> 7) * (kWgPos * 128) + (kl & 127));
            const uint64_t bh = desc_sw128(sb + (kh >> 7) * (32 * 128) + (kh & 127));
            const uint64_t bl = desc_sw128(sb + (kl >> 7) * (32 * 128) + (kl & 127));
            mma_m64n32_ss(d[s], ah, bh, ks > 0);
            mma_m64n32_ss(d[s], al, bh, 1);
            mma_m64n32_ss(d[s], ah, bl, 1);
          }
        }
        mma_commit();
        // item k + 1's gathers fly under the MMAs: its buffer's last reader finished before the closing barrier
        // of item k - 1; the ids of item k + 2 are requested behind them
        gather(k + 1, ids_next);
        cp_async_commit();
        load_ids(k + 2, ids_next);
        clk.lap(PH_GATHER_ISSUE);
        mma_wait<0>();
  #pragma unroll
        for (int s = 0; s < R; ++s) reg_fence(d[s]);
      }
      clk.lap(PH_AU_MMA);
      // ---- gate: positions pr = 16 warp + g + 8 h; the quad of lanes sharing a position sums its 32 units
  #pragma unroll
      for (int s = 0; s < R; ++s) {
        if (!live[s]) continue;
  #pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int pr = 16 * warp + g + 8 * h;
          float acc = 0.f;
  #pragma unroll
          for (int j = 0; j < 4; ++j)
  #pragma unroll
            for (int c = 0; c < 2; ++c) {
              const float z = d[s][4 * j + 2 * h + c] + cstv[s][2 * j + c];
              acc = fmaf(z, z > 0.f ? wout[2 * j + c] : slope[h][2 * j + c], acc);
            }
          acc += __shfl_xor_sync(0xffffffffu, acc, 1);
          acc += __shfl_xor_sync(0xffffffffu, acc, 2);
          // w split to bf16 hi / lo into rows 0 and 1 of the row's pooling operand (K byte 2 pr); w = 0 past nt
          const float w = pr < nt ? rcp_approx(1.f + __expf(-(acc + p.au_bout))) : 0.f;
          if (cq == 0) {
            const uint32_t pb = pb_s + s * L::PB_BYTES;
            const __nv_bfloat16 wh16 = __float2bfloat16_rn(w);
            const __nv_bfloat16 wl16 = __float2bfloat16_rn(w - __bfloat162float(wh16));
            st_shared_u16(pb + sw128_offset(0, pr >> 3) + 2 * (pr & 7), __bfloat16_as_ushort(wh16));
            st_shared_u16(pb + sw128_offset(1, pr >> 3) + 2 * (pr & 7), __bfloat16_as_ushort(wl16));
          }
        }
      }
      fence_async_smem();
      named_sync(1 + q, 128);                                 // w in place
      clk.lap(PH_GATE);
      // ---- pooling: D (+)= A^T Pb over the tile's 64 positions, A read MN-major (its 128-byte rows are
      // positions); products h_hi w_hi, h_lo w_hi, h_hi w_lo as in the activation unit; the rows' MMAs in one
      // commit group
      {
        // (an accumulator set that stayed live across the next activation-unit MMAs would make ptxas spill)
        float pd[R][KB][4];
        mma_fence();
  #pragma unroll
        for (int s = 0; s < R; ++s) {
          const uint32_t as = live[s] ? sa + s * L::A_BYTES : sa, ps = live[s] ? pb_s + s * L::PB_BYTES : pb_s;
  #pragma unroll
          for (int ks = 0; ks < kWgPos / 16; ++ks)
  #pragma unroll
            for (int kb = 0; kb < KB; ++kb)
              mma_m64n8_ss_amn(pd[s][kb], desc_sw128_mn(as + kb * (kWgPos * 128) + ks * 2048),
                               desc_sw128(ps + 32 * ks), ks > 0);
        }
        mma_commit();
        // the next row's W_r and gate constants under the MMAs: every warp of the warpgroup has waited for this
        // row's activation-unit MMAs (the gate barrier) and used its gate constants
        if (k + 1 < n_items && item_ch(k + 1) == 0) build_wr(k + 1);
        clk.lap(PH_W_BUILD);
        mma_wait<0>();
  #pragma unroll
        for (int s = 0; s < R; ++s) {
          if (!live[s]) continue;
  #pragma unroll
          for (int kb = 0; kb < KB; ++kb) {
            reg_fence(pd[s][kb]);
  #pragma unroll
            for (int e = 0; e < 4; ++e) pacc[s][kb][e] = ch > 0 ? pacc[s][kb][e] + pd[s][kb][e] : pd[s][kb][e];
          }
        }
      }
      // lanes cq = 0 hold columns w hi (pacc[s][.][0], [2]) and w lo ([1], [3]) of operand columns 16 warp + g (+ 8);
      // at EP = 32 the lo elements' sums (columns 32 + e) are in warps 2 and 3 and go through shared memory
      const bool last = ch == nch - 1;
      if (EP == 32 && last && warp >= 2 && cq == 0) {
  #pragma unroll
        for (int s = 0; s < R; ++s) {
          if (!live[s]) continue;
          pool_lo[32 * s + 16 * (warp - 2) + g] = pacc[s][0][0];
          pool_lo[32 * s + 16 * (warp - 2) + g + 8] = pacc[s][0][2];
        }
      }
      named_sync(1 + q, 128);                                 // tiles of item k, Pb and W_r free again
      if (last && cq == 0 && (EP == 64 || warp < 2)) {
  #pragma unroll
        for (int s = 0; s < R; ++s) {
          if (!live[s]) continue;
          float* xrow = Xs + r[s] * L::LDX;
  #pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int e = 16 * warp + g + 8 * h;
            const float lo_whi = EP == 32 ? pool_lo[32 * s + e] : pacc[s][KB - 1][2 * h];
            xrow[OFF_POOL + e] = (pacc[s][0][2 * h] + lo_whi) + pacc[s][0][2 * h + 1];
          }
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
        // (W1^T's part first: Dense(128) waits for it, Dense(64) for W2^T's)
        fence_async_smem();
        if (L::RELOAD_W1 > 0) {
          mbar_arrive_expect_tx(&reload_bar[0], L::RELOAD_W1);
          for (uint32_t off = L::IMG_RESIDENT; off < L::RELOAD_W2_OFF; off += 32768u)
            bulk_g2s(img + off, p.mlp_image + off, min(32768u, L::RELOAD_W2_OFF - off), &reload_bar[0]);
        }
        if (L::RELOAD_W2 > 0) {
          mbar_arrive_expect_tx(&reload_bar[1], L::RELOAD_W2);
          for (uint32_t off = L::RELOAD_W2_OFF; off < L::IMG_BYTES; off += 32768u)
            bulk_g2s(img + off, p.mlp_image + off, min(32768u, L::IMG_BYTES - off), &reload_bar[1]);
        }
      }
      top_mlp_wg<EP>(p, b, row0, Xs, base + L::OPS_OFF, img, fs + L::F_RED, weights_ready ? nullptr : &res_bar,
                     reload_bar, reload_parity, clk);
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
