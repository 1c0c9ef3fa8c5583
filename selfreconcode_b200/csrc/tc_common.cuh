// Shared pieces of the tensor-core engine (tc_gemm.cu: layer GEMMs, tc_wgrad.cu: weight-gradient GEMMs):
// tile geometry of the pre-tiled split-bf16 operands, Hopper wgmma wrappers.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace sr_tc {

#ifndef SR_TC_PLANES
#define SR_TC_PLANES 2
#endif
constexpr int kPlanes = SR_TC_PLANES;
// BN = the column tile of a layer launch; layers with N <= BN_NARROW run (and their weights are packed) on the
// narrow tile instead (tile_n)
constexpr int BM = 128, BN = 256, BN_NARROW = 64, BK = 32, STAGES = kPlanes == 2 ? 3 : 2;
constexpr int A_PLANE = BM * BK;          // elements
constexpr int A_STAGE = kPlanes * A_PLANE;   // 2 planes: 16 KB
constexpr uint32_t A_STAGE_BYTES = A_STAGE * 2;
__host__ __device__ constexpr int tile_n(int N) { return N <= BN_NARROW ? BN_NARROW : BN; }

// ---- tiled ("pre-swizzled") global layouts ----------------------------------------------------
// A: [row tile mt][k chunk kc][plane p][k8 (4)][row group (16)][row (8)][elem (8)]
// W: [col tile nt][k chunk kc][plane p][k8 (4)][row group (bn / 8)][row (8)][elem (8)], bn = tile_n(N)
__host__ __device__ inline size_t a_tile_off(long long mt, int kc, int KC, int p) {
  return (((size_t)mt * KC + kc) * kPlanes + p) * A_PLANE;
}
__host__ __device__ inline size_t w_tile_off(int bn, int nt, int kc, int KC, int p) {
  return (((size_t)nt * KC + kc) * kPlanes + p) * (size_t)(bn * BK);
}
__device__ __forceinline__ int in_tile_off(int rows_per_tile, int r, int k) {
  return (k >> 3) * (rows_per_tile * 8) + (r >> 3) * 64 + (r & 7) * 8 + (k & 7);
}

__device__ __forceinline__ void split3(float x, __nv_bfloat16& b1, __nv_bfloat16& b2, __nv_bfloat16& b3) {
  b1 = __float2bfloat16_rn(x);
  const float r1 = x - __bfloat162float(b1);
  b2 = __float2bfloat16_rn(r1);
  const float r2 = r1 - __bfloat162float(b2);
  b3 = __float2bfloat16_rn(r2);
}

// ---- wgmma wrappers (sm_90a) ------------------------------------------------------------------
// Shared-memory matrix descriptor, no swizzle: start[0,14) lbo[16,30) sbo[32,46) (all >> 4).
// LBO = byte stride between adjacent 8x8 core matrices along K, SBO = along M / N.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Named barrier over the 128 threads of one warpgroup (ids 1.. ; 0 is __syncthreads).
__device__ __forceinline__ void warpgroup_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

#define SR_ACC8(c, d, i)                                                                                \
  c(d[i]), c(d[i + 1]), c(d[i + 2]), c(d[i + 3]), c(d[i + 4]), c(d[i + 5]), c(d[i + 6]), c(d[i + 7])
#define SR_ACC32(c, d, i) SR_ACC8(c, d, i), SR_ACC8(c, d, i + 8), SR_ACC8(c, d, i + 16), SR_ACC8(c, d, i + 24)
#define SR_ACC128(c, d) SR_ACC32(c, d, 0), SR_ACC32(c, d, 32), SR_ACC32(c, d, 64), SR_ACC32(c, d, 96)
#define SR_WGMMA_M64N256K16_BF16                                                                                   \
  "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"                                                            \
  "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "                                                         \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "     \
  "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "      \
  "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "      \
  "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, "      \
  "%86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, "     \
  "%106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, "   \
  "%124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}\n"

// D[64 x 256] (fp32, registers of the warpgroup) (+)= A[64 x 16] * B[16 x 256], both bf16 from shared memory.
// TA / TB = 1: the operand is MN-major (transposed) in shared memory.  FIRST: D = A * B, the old accumulator is
// neither read nor kept live (write-only register operands).  Fragment of thread t (warp w = t / 32 of the
// warpgroup, lane l): d[4 i + {0, 1}] = row 16 w + l / 4, columns 8 i + 2 (l % 4) + {0, 1}; d[4 i + {2, 3}]: row + 8.
#define SR_OUT(x) "=f"(x)
#define SR_INOUT(x) "+f"(x)
template <int TA, int TB, bool FIRST>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t adesc, uint64_t bdesc) {
  if constexpr (FIRST)
    asm volatile(SR_WGMMA_M64N256K16_BF16
                 : SR_ACC128(SR_OUT, d)
                 : "l"(adesc), "l"(bdesc), "r"(0), "n"(TA), "n"(TB));
  else
    asm volatile(SR_WGMMA_M64N256K16_BF16
                 : SR_ACC128(SR_INOUT, d)
                 : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA), "n"(TB));
}
#define SR_WGMMA_M64N64K16_BF16                                                                                    \
  "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                                             \
  "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "                                                          \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "     \
  "%23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
// The same for a 64-column tile: d[32], the fragment as above with i < 8.
template <int TA, int TB, bool FIRST>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  if constexpr (FIRST)
    asm volatile(SR_WGMMA_M64N64K16_BF16
                 : SR_ACC32(SR_OUT, d, 0)
                 : "l"(adesc), "l"(bdesc), "r"(0), "n"(TA), "n"(TB));
  else
    asm volatile(SR_WGMMA_M64N64K16_BF16
                 : SR_ACC32(SR_INOUT, d, 0)
                 : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA), "n"(TB));
}
#undef SR_OUT
#undef SR_INOUT
#undef SR_WGMMA_M64N64K16_BF16
#undef SR_WGMMA_M64N256K16_BF16
#undef SR_ACC128
#undef SR_ACC32
#undef SR_ACC8

}  // namespace sr_tc
