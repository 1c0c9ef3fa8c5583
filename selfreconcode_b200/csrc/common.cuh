// Shared device/host helpers for the selfrecon-b200 kernels (sm_90a: H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/selfrecon_b200.h"

#define SR_NUM_SMS 132   // H100 SXM

// Launch-error -> C-ABI return code. Never synchronises.
static inline int sr_launch_status() {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();
    return (int)e;
  }
  return SR_OK;
}

static inline int sr_div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Grid sized as a multiple of the SM count (persistent / grid-stride kernels).
static inline int sr_grid_for(long long n, int threads, int ctas_per_sm) {
  long long need = (n + threads - 1) / threads;
  long long cap = (long long)SR_NUM_SMS * ctas_per_sm;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------------
// mbarrier + bulk-async-copy (TMA engine, 1-D form: SASS UBLKCP) wrappers.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sr_smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void sr_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sr_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void sr_fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void sr_fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void sr_mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sr_smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void sr_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(sr_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void sr_mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra.uni WAIT_DONE;\n"
      "bra.uni WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(sr_smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy, completion signalled on an mbarrier (bytes multiple of 16).
__device__ __forceinline__ void sr_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          sr_smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(sr_smem_u32(bar))
      : "memory");
}

__device__ __forceinline__ float sr_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int sr_warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif
