// wgmma_selftest.cu - one-CTA known-answer kernel for the warpgroup-MMA plumbing in wgmma.cuh:
// operand layouts (SW128 K-major smem tiles, A fragments in registers), descriptors, accumulator
// fragment layout.  D[128][N] = bf16(A)[128][K] * bf16(B)[N][K]^T with fp32 accumulate, as two
// M = 64 halves issued by one warpgroup.  N = 8: A is stored MN-major (each 128-byte row holds 64 M values of
// one k, as din_wg_kernel's pooling reads its history tiles) and read through desc_sw128_mn.
// Exposed as srs_selftest_wgmma (include/srs_ctr.h) and checked by tests/test_gpu_umma.py.
#include "kernels.h"
#include "wgmma.cuh"

namespace srs {
using namespace wg;

template <int N>
__device__ __forceinline__ void selftest_half(const float* __restrict__ A, float* __restrict__ D, int K, int KB,
                                              int a_in_regs, uint32_t sA, uint32_t sB, int half) {
  constexpr int NR = N / 2;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, cq = lane & 3;
  float d[NR];
#pragma unroll
  for (int i = 0; i < NR; ++i) d[i] = 0.f;
  mma_fence();
  for (int kb = 0; kb < KB; ++kb)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t bd = desc_sw128(sB + kb * (N * 128)) + 2 * ks;
      const int acc = kb > 0 || ks > 0;
      if (N != 8 && a_in_regs) {
        // m64k16 A fragment: rows 16 w + g (+8), k = 2 cq (+1), 2 cq + 8 (+9) of this K step
        const int r0 = 64 * half + 16 * warp + g, k0 = kb * 64 + ks * 16 + 2 * cq;
        const float* a0 = A + (size_t)r0 * K + k0;
        const float* a1 = A + (size_t)(r0 + 8) * K + k0;
        const uint32_t a[4] = {pack_hi(a0[0], a0[1]), pack_hi(a1[0], a1[1]), pack_hi(a0[8], a0[9]),
                               pack_hi(a1[8], a1[9])};
        if constexpr (N == 32) mma_m64n32_rs(d, a, bd, acc);
        else if constexpr (N == 16) mma_m64n16_rs(d, a, bd, acc);
      } else if constexpr (N == 8) {
        // MN-major: half h holds K rows of its 64 M values; one K = 16 step is 16 rows
        const uint64_t ad = desc_sw128_mn(sA + half * (K * 128) + (kb * 4 + ks) * 2048);
        mma_m64n8_ss_amn(d, ad, bd, acc);
      } else {
        const uint64_t ad = desc_sw128(sA + kb * 16384 + half * 8192) + 2 * ks;
        if constexpr (N == 32) mma_m64n32_ss(d, ad, bd, acc);
        else mma_m64n16_ss(d, ad, bd, acc);
      }
    }
  mma_commit();
  mma_wait<0>();
  reg_fence(d);
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c)
        D[(size_t)(64 * half + 16 * warp + g + 8 * i) * N + 8 * j + 2 * cq + c] = d[4 * j + 2 * i + c];
}

__global__ void __launch_bounds__(128) wgmma_selftest_kernel(const float* __restrict__ A,
                                                             const float* __restrict__ Bm,
                                                             float* __restrict__ D, int N, int KB,
                                                             int a_in_regs) {
  extern __shared__ uint8_t raw[];
  const int tid = threadIdx.x;
  const int K = KB * 64;
  uint8_t* base = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
  uint8_t* sA = base;                          // KB tiles of 128 rows x 128 B
  uint8_t* sB = base + KB * 16384;             // KB tiles of N rows x 128 B (1024-aligned)
  for (int kb = 0; kb < KB; ++kb) {
    const float* arow = A + (size_t)tid * K + kb * 64;
#pragma unroll
    for (int c = 0; c < 8 * (N != 8); ++c) {
      uint4 v;
      v.x = pack_hi(arow[8 * c + 0], arow[8 * c + 1]);
      v.y = pack_hi(arow[8 * c + 2], arow[8 * c + 3]);
      v.z = pack_hi(arow[8 * c + 4], arow[8 * c + 5]);
      v.w = pack_hi(arow[8 * c + 6], arow[8 * c + 7]);
      *reinterpret_cast<uint4*>(sA + kb * 16384 + sw128_offset(tid, c)) = v;
    }
    if (tid < N) {
      const float* brow = Bm + (size_t)tid * K + kb * 64;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        uint4 v;
        v.x = pack_hi(brow[8 * c + 0], brow[8 * c + 1]);
        v.y = pack_hi(brow[8 * c + 2], brow[8 * c + 3]);
        v.z = pack_hi(brow[8 * c + 4], brow[8 * c + 5]);
        v.w = pack_hi(brow[8 * c + 6], brow[8 * c + 7]);
        *reinterpret_cast<uint4*>(sB + kb * (N * 128) + sw128_offset(tid, c)) = v;
      }
    }
  }
  if (N == 8) {                               // A MN-major: row k of half h = A[64 h .. 64 h + 63][k]
    for (int i = tid; i < 2 * K; i += 128) {
      const int half = i / K, k = i % K;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float* a = A + (size_t)(64 * half + 8 * c) * K + k;
        uint4 v;
        v.x = pack_hi(a[0], a[K]);
        v.y = pack_hi(a[2 * K], a[3 * K]);
        v.z = pack_hi(a[4 * K], a[5 * K]);
        v.w = pack_hi(a[6 * K], a[7 * K]);
        *reinterpret_cast<uint4*>(sA + half * (K * 128) + sw128_offset(k, c)) = v;
      }
    }
  }
  fence_async_smem();
  __syncthreads();
  for (int half = 0; half < 2; ++half) {
    if (N == 8) selftest_half<8>(A, D, K, KB, a_in_regs, smem_u32(sA), smem_u32(sB), half);
    else if (N == 32) selftest_half<32>(A, D, K, KB, a_in_regs, smem_u32(sA), smem_u32(sB), half);
    else selftest_half<16>(A, D, K, KB, a_in_regs, smem_u32(sA), smem_u32(sB), half);
  }
}

cudaError_t launch_wgmma_selftest(const float* A, const float* B, float* D, int N, int KB, int a_in_regs,
                                  cudaStream_t s) {
  if ((N != 8 && N != 16 && N != 32) || KB < 1 || KB > 4 || (N == 8 && a_in_regs)) return cudaErrorInvalidValue;
  const size_t smem = 1024 + (size_t)KB * 16384 + (size_t)KB * N * 128;
  cudaError_t e = cudaFuncSetAttribute(wgmma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  wgmma_selftest_kernel<<<1, 128, smem, s>>>(A, B, D, N, KB, a_in_regs);
  ++g_launch_count;
  return cudaGetLastError();
}

}  // namespace srs
