// wgmma.cuh - hand-written sm_90a building blocks: warpgroup MMA (wgmma.mma_async) wrappers,
// the shared-memory matrix descriptor for K-major 128-byte-swizzled bf16 tiles, proxy fences,
// cp.async and the bf16 hi/lo split.
//
// Layout conventions used by every kernel that includes this file:
//   * an operand tile is stored K-major in 128-byte rows (64 bf16), 8-row groups of 1024 bytes,
//     the 16-byte chunk index of each row XOR-ed with (row & 7) (SWIZZLE_128B).  Tiles are
//     1024-byte aligned.  K > 64 is a sequence of such tiles ("K blocks").
//   * one wgmma (bf16 x bf16 -> f32) consumes K = 16 elements = 32 bytes of each row; successive
//     K steps inside a K block advance the descriptor start address by 32 bytes.
//   * accumulators of m64nNk16 live in the registers of the issuing warpgroup: register
//     4 j + 2 i + c of thread (warp w, lane l) holds D[16 w + l / 4 + 8 i][8 j + 2 (l % 4) + c].
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace srs {
namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void st_shared_u32(uint32_t smem_addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(smem_addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_shared_u16(uint32_t smem_addr, unsigned short v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(smem_addr), "h"(v) : "memory");
}

// byte offset of (row, 16-byte chunk c) inside a SW128 K-major tile
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk) {
  return row * 128u + ((chunk ^ (row & 7u)) << 4);
}

// wgmma shared-memory matrix descriptor: K-major, SWIZZLE_128B, 8-row groups 1024 B apart.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t smem_addr_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr_bytes & 0x3FFFF) >> 4);   // start address
  d |= (uint64_t)1 << 16;                               // leading byte offset (unused for SW128 K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                     // stride byte offset: 8 rows * 128 B
  d |= (uint64_t)1 << 62;                               // SWIZZLE_128B
  return d;
}

// wgmma shared-memory matrix descriptor: MN-major, SWIZZLE_128B.  Each 128-byte row holds 64 consecutive
// M (or N) elements of one K index, rows swizzled as in a K-major tile, so a K-major tile read this way is its
// own transpose.  Stride byte offset: 8 K rows (1024 B) to the next 8; leading byte offset: one 64-element MN
// block to the next, never reached by a 64-wide operand.  One K = 16 step advances the start by 2048 B.
__device__ __forceinline__ uint64_t desc_sw128_mn(uint32_t smem_addr_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr_bytes & 0x3FFFF) >> 4);   // start address
  d |= (uint64_t)(1024 >> 4) << 16;                     // leading byte offset (unused at 64 MN elements)
  d |= (uint64_t)(1024 >> 4) << 32;                     // stride byte offset: 8 K rows * 128 B
  d |= (uint64_t)1 << 62;                               // SWIZZLE_128B
  return d;
}

// generic-proxy writes (st.shared, cp.async) -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void mma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void mma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// the accumulator registers are written asynchronously: keep the compiler from moving their uses
// across the wait
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- warpgroup MMAs, bf16 x bf16 -> f32, B K-major from shared memory ---------------------------
// D[64 x 32] (+)= A[smem desc] * B[smem desc]
__device__ __forceinline__ void mma_m64n32_ss(float (&d)[16], uint64_t a, uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(accumulate));
}
// D[64 x 32] (+)= A[registers] * B[smem desc]
__device__ __forceinline__ void mma_m64n32_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate));
}
// D[64 x 16] (+)= A[smem desc] * B[smem desc]
__device__ __forceinline__ void mma_m64n16_ss(float (&d)[8], uint64_t a, uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(accumulate));
}
// D[64 x 16] (+)= A[registers] * B[smem desc]
__device__ __forceinline__ void mma_m64n16_rs(float (&d)[8], const uint32_t (&a)[4], uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate));
}
// D[64 x 8] (+)= A[smem desc, MN-major: desc_sw128_mn] * B[smem desc, K-major]
__device__ __forceinline__ void mma_m64n8_ss_amn(float (&d)[4], uint64_t a, uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3}, %4, %5, p, 1, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(a), "l"(b), "r"(accumulate));
}

// D[64 x 64] (+)= A[smem desc] * B[smem desc]
__device__ __forceinline__ void mma_m64n64_ss(float (&d)[32], uint64_t a, uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(accumulate));
}
// D[64 x 128] (+)= A[smem desc] * B[smem desc]
__device__ __forceinline__ void mma_m64n128_ss(float (&d)[64], uint64_t a, uint64_t b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(accumulate));
}

// ---- mbarrier and bulk async copy global -> shared (TMA engine, no tensor map) ------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// brings the line holding p into L1 (and L2); no register waits for it
__device__ __forceinline__ void prefetch_l1(const void* p) {
  asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
}
// read-only load that allocates no L1 line (L1::no_allocate): for a stream read once, so that it does not
// evict the rows that cp_async16_zfill finds in L1
__device__ __forceinline__ int ldg_stream(const int* p) {
  int v;
  asm("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

// ---- cp.async, named barriers --------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// copies the first src_bytes (0 or 16) of src and zero-fills the rest of the 16 bytes; 0 reads nothing.
// The source goes through L1 (.ca): the embedding rows it copies are gathered by id, and a few ids (the
// padding row, popular movies) recur across a CTA's tiles, so a row read once is served from L1 after that
// instead of queueing with every other SM on the same L2 line.  L1 is not coherent with other SMs' writes:
// this is valid because no predict launch writes a table that it gathers.
__device__ __forceinline__ void cp_async16_zfill(void* dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void named_sync(int id, int n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}

// ---- bf16 hi/lo split ("bf16x3": x*w ~ hi*whi + lo*whi + hi*wlo) ------------------------------
// hi = x rounded to bf16 (round-to-nearest-even), lo = (x - hi) rounded to bf16; x - hi is
// exact in fp32 and |x - hi - lo| <= 2^-17 |x|.
struct Split2 {
  uint32_t hi, lo;      // packed pairs: first value in the low half
};
__device__ __forceinline__ Split2 split_pack(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const uint32_t hb = *reinterpret_cast<uint32_t*>(&h);
  __nv_bfloat162 l = __floats2bfloat162_rn(a - __uint_as_float(hb << 16), b - __uint_as_float(hb & 0xFFFF0000u));
  Split2 r;
  r.hi = hb;
  r.lo = *reinterpret_cast<uint32_t*>(&l);
  return r;
}
// truncating variant used by the self test (exactly representable operands)
__device__ __forceinline__ uint32_t pack_hi(float a, float b) {   // (a -> low half, b -> high half)
  return __byte_perm(__float_as_uint(a), __float_as_uint(b), 0x7632);
}

}  // namespace wg
}  // namespace srs
