// Batched 3x3 inverse and its analytic VJP (SURVEY.md rows a14 / K1 / K2).
//
// Semantics follow FastMinv/Matrix3x3InvKernels.cu:22-104 of the reference:
//   inv = adj(m)/det ; if |det| < 1e-4 (compared in double) -> inv = 0, check = false
//   backward: out = -(C^T G C^T) with C = inv.
//
// Notes: the op is a pure HBM stream (73 B / matrix forward, 108 B backward), so the
// kernel stages each CTA's contiguous [256 x 9] block through shared memory to turn the
// stride-9 per-thread accesses of the reference into fully coalesced 128-bit global
// transactions; the grid is a multiple of the SM count with a grid-stride loop.
#include "common.cuh"
#include "trace_rules.cuh"

namespace {

constexpr int kThreads = 256;

template <typename T>
__device__ __forceinline__ void load_tile(const T* __restrict__ g, T* s, int64_t base, int64_t n,
                                          int tid) {
  // contiguous [cnt*9] elements
  int64_t rem = n - base;
  int cnt = rem < kThreads ? (int)rem : kThreads;
  const T* src = g + base * 9;
  for (int i = tid; i < cnt * 9; i += kThreads) s[i] = src[i];
}

template <typename T>
__device__ __forceinline__ void store_tile(T* __restrict__ g, const T* s, int64_t base, int64_t n,
                                           int tid) {
  int64_t rem = n - base;
  int cnt = rem < kThreads ? (int)rem : kThreads;
  T* dst = g + base * 9;
  for (int i = tid; i < cnt * 9; i += kThreads) dst[i] = s[i];
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
minv3x3_kernel(const T* __restrict__ ms, T* __restrict__ invs, uint8_t* __restrict__ checks,
               int64_t n) {
  __shared__ T sm[kThreads * 9];
  const int tid = threadIdx.x;
  for (int64_t base = (int64_t)blockIdx.x * kThreads; base < n;
       base += (int64_t)gridDim.x * kThreads) {
    load_tile(ms, sm, base, n, tid);
    __syncthreads();
    int64_t mid = base + tid;
    if (mid < n) {
      T m[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) m[i] = sm[tid * 9 + i];  // stride 9: conflict free (9 odd)
      T c[9], det, o[9];
      const bool ok = minv3x3_cofactors(m, c, det);
      if (ok) {
#pragma unroll
        for (int i = 0; i < 9; ++i) o[i] = c[3 * (i % 3) + i / 3] / det;  // o[r][k] = c[k][r] / det
      } else {
#pragma unroll
        for (int i = 0; i < 9; ++i) o[i] = T(0);
      }
#pragma unroll
      for (int i = 0; i < 9; ++i) sm[tid * 9 + i] = o[i];
      checks[mid] = ok ? 1 : 0;
    }
    __syncthreads();
    store_tile(invs, sm, base, n, tid);
    __syncthreads();
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
minv3x3_bwd_kernel(const T* __restrict__ grads, const T* __restrict__ invs, T* __restrict__ outs,
                   int64_t n) {
  __shared__ T sg[kThreads * 9];
  __shared__ T sc[kThreads * 9];
  const int tid = threadIdx.x;
  for (int64_t base = (int64_t)blockIdx.x * kThreads; base < n;
       base += (int64_t)gridDim.x * kThreads) {
    load_tile(grads, sg, base, n, tid);
    load_tile(invs, sc, base, n, tid);
    __syncthreads();
    if (base + tid < n) {
      T g[9], c[9], o[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        g[i] = sg[tid * 9 + i];
        c[i] = sc[tid * 9 + i];
      }
      // out[a][b] = - sum_{i,j} g[i][j] * c[i][a] * c[b][j]   ( = -(C^T G C^T)[a][b] ),
      // accumulated in the (i,j) row-major order of the reference's explicit 9-term sums.
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) {
          T acc = T(0);
#pragma unroll
          for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) {
              T term = g[3 * i + j] * c[3 * i + a] * c[3 * b + j];
              acc = (i == 0 && j == 0) ? term : acc + term;
            }
          o[3 * a + b] = -acc;
        }
#pragma unroll
      for (int i = 0; i < 9; ++i) sg[tid * 9 + i] = o[i];
    }
    __syncthreads();
    store_tile(outs, sg, base, n, tid);
    __syncthreads();
  }
}

template <typename T>
int launch_fwd(const T* ms, T* invs, uint8_t* checks, int64_t n, cudaStream_t s) {
  if (n < 0) return SR_EINVAL;
  if (n == 0) return SR_OK;
  if (!ms || !invs || !checks) return SR_EINVAL;
  int grid = sr_grid_for(n, kThreads, 8);
  minv3x3_kernel<T><<<grid, kThreads, 0, s>>>(ms, invs, checks, n);
  return sr_launch_status();
}
template <typename T>
int launch_bwd(const T* g, const T* c, T* o, int64_t n, cudaStream_t s) {
  if (n < 0) return SR_EINVAL;
  if (n == 0) return SR_OK;
  if (!g || !c || !o) return SR_EINVAL;
  int grid = sr_grid_for(n, kThreads, 8);
  minv3x3_bwd_kernel<T><<<grid, kThreads, 0, s>>>(g, c, o, n);
  return sr_launch_status();
}

}  // namespace

extern "C" {
int sr_minv3x3_f32(const float* ms, float* invs, uint8_t* checks, int64_t n, cudaStream_t s) {
  return launch_fwd<float>(ms, invs, checks, n, s);
}
int sr_minv3x3_f64(const double* ms, double* invs, uint8_t* checks, int64_t n, cudaStream_t s) {
  return launch_fwd<double>(ms, invs, checks, n, s);
}
int sr_minv3x3_bwd_f32(const float* g, const float* c, float* o, int64_t n, cudaStream_t s) {
  return launch_bwd<float>(g, c, o, n, s);
}
int sr_minv3x3_bwd_f64(const double* g, const double* c, double* o, int64_t n, cudaStream_t s) {
  return launch_bwd<double>(g, c, o, n, s);
}
}
