// 3-D trilinear grid sampler, border padding, align_corners=False, with first- and
// second-order backward (SURVEY.md rows a6 / K7-K9).
//
// Semantics follow MCAcc/cuda/GridSamplerMineKernel.cu:160-914 of the reference:
//   un-normalise   x -> ((x + 1.f) * W - 1.) / 2.   (float add/mul, then double, :210-212; for
//                  double input the product is rounded before the subtraction, never fused)
//   border clip    min(W-1, max(x, 0)); gradient multiplier 0 when x<=0 or x>=W-1 (:33-61).
//                  A NaN coordinate is sampled at 0 with multiplier 0, so its backward is the gradient of
//                  what the forward computed (the reference samples it at 0 but sends its grad_input to
//                  no voxel; the grid gradient is 0 either way)
//   corners        floor(x) and +1; out-of-range corners are skipped (their weight is 0)
//   forward        8 corners accumulated x-fastest, y, z with one FMA each (:285-309)
//   backward       grad_input by atomicAdd, grad_grid scaled by W/2 and the border mask
//   dbackward      gradients of (grad_input, grad_grid) wrt input, grid and grad_output,
//                  including the mixed second derivatives of the trilinear weights (:688-855)
//
// Layout: `input` may have arbitrary strides (the reference passes the NCDHW skin-weight
// volume); grid is [N,P,3], output/grad_output are [N,C,P].  One thread per sample point,
// channel loop inside (the three grid gradients are reductions over channels).  The op is
// gather-bound: 8 corners x C channels x 4 B per point; the fused LBS path in lbs.cu uses a
// channels-last copy of the volume instead and does not go through this kernel.
#include "common.cuh"

namespace {

constexpr int kThreads = 128;

template <typename T>
struct Axis {
  int i0;    // floor of the clipped coordinate
  T a[2];    // weights towards corner i0 / i0+1
  T mult;    // border mask for the coordinate gradient (0 or 1)
  bool in0, in1;
};

__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }

template <typename T>
__device__ __forceinline__ Axis<T> make_axis(T g, int size) {
  Axis<T> ax;
  // ((g + 1.f) * size - 1.) / 2.   with the reference's mixed precision.  The product is rounded to T
  // before the subtraction in both precisions: in double the compiler would otherwise fuse
  // `prod - 1.0` into an FMA, and x would differ by an ulp, enough to move floor(x) at a voxel face.
  T prod = mul_rn(g + (T)1, (T)size);
  T x = (T)(((double)prod - 1.0) / 2.0);
  const T hi = (T)(size - 1);
  if (!(x > (T)0)) {  // x <= 0 (or NaN)
    ax.mult = (T)0;
    x = (T)0;
  } else if (x >= hi) {
    ax.mult = (T)0;
    x = hi;
  } else {
    ax.mult = (T)1;
  }
  const int i0 = (int)floor((double)x);
  ax.i0 = i0;
  ax.a[0] = (T)(i0 + 1) - x;
  ax.a[1] = x - (T)i0;
  ax.in0 = i0 >= 0 && i0 < size;
  ax.in1 = (i0 + 1) >= 0 && (i0 + 1) < size;
  return ax;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
gs3d_fwd_kernel(const T* __restrict__ input, long long sN, long long sC, long long sD,
                long long sH, long long sW, const T* __restrict__ grid, T* __restrict__ output,
                int32_t* __restrict__ corner_idx, int N, int C, int D, int H, int W, long long P) {
  const long long total = (long long)N * P;
  for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * kThreads) {
    const long long n = idx / P, p = idx - n * P;
    const T* g = grid + idx * 3;
    const Axis<T> ax = make_axis<T>(g[0], W), ay = make_axis<T>(g[1], H),
                  az = make_axis<T>(g[2], D);
    if (corner_idx) {
      corner_idx[idx * 3 + 0] = ax.i0;
      corner_idx[idx * 3 + 1] = ay.i0;
      corner_idx[idx * 3 + 2] = az.i0;
    }
    T w[8];
    long long off[8];
    bool ok[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int bx = k & 1, by = (k >> 1) & 1, bz = k >> 2;
      w[k] = ax.a[bx] * ay.a[by] * az.a[bz];
      ok[k] = (bx ? ax.in1 : ax.in0) && (by ? ay.in1 : ay.in0) && (bz ? az.in1 : az.in0);
      off[k] = (long long)(az.i0 + bz) * sD + (long long)(ay.i0 + by) * sH +
               (long long)(ax.i0 + bx) * sW;
    }
    const T* base = input + n * sN;
    T* out = output + n * (long long)C * P + p;
    for (int c = 0; c < C; ++c, base += sC, out += P) {
      T acc = (T)0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (ok[k]) acc = fma(__ldg(base + off[k]), w[k], acc);
      *out = acc;
    }
  }
}

__device__ __forceinline__ void atomic_add(float* p, float v) { atomicAdd(p, v); }
__device__ __forceinline__ void atomic_add(double* p, double v) { atomicAdd(p, v); }

template <typename T>
__global__ void __launch_bounds__(kThreads)
gs3d_bwd_kernel(const T* __restrict__ input, long long sN, long long sC, long long sD,
                long long sH, long long sW, const T* __restrict__ grid,
                const T* __restrict__ gout, T* __restrict__ ginp, T* __restrict__ ggrid, int N,
                int C, int D, int H, int W, long long P) {
  const long long total = (long long)N * P;
  const long long cD = (long long)H * W, cC = (long long)D * H * W;  // contiguous grad_input
  for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * kThreads) {
    const long long n = idx / P, p = idx - n * P;
    const T* g = grid + idx * 3;
    const Axis<T> ax = make_axis<T>(g[0], W), ay = make_axis<T>(g[1], H),
                  az = make_axis<T>(g[2], D);
    T w[8], dx[8], dy[8], dz[8];
    long long off[8], coff[8];
    bool ok[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int bx = k & 1, by = (k >> 1) & 1, bz = k >> 2;
      const T sx = bx ? (T)1 : (T)-1, sy = by ? (T)1 : (T)-1, sz = bz ? (T)1 : (T)-1;
      w[k] = ax.a[bx] * ay.a[by] * az.a[bz];
      dx[k] = sx * ay.a[by] * az.a[bz];
      dy[k] = sy * ax.a[bx] * az.a[bz];
      dz[k] = sz * ax.a[bx] * ay.a[by];
      ok[k] = (bx ? ax.in1 : ax.in0) && (by ? ay.in1 : ay.in0) && (bz ? az.in1 : az.in0);
      off[k] = (long long)(az.i0 + bz) * sD + (long long)(ay.i0 + by) * sH +
               (long long)(ax.i0 + bx) * sW;
      coff[k] = (long long)(az.i0 + bz) * cD + (long long)(ay.i0 + by) * W + (ax.i0 + bx);
    }
    const T* base = input + n * sN;
    T* gi = ginp + n * (long long)C * cC;
    const T* go = gout + n * (long long)C * P + p;
    T gix = (T)0, giy = (T)0, giz = (T)0;
    for (int c = 0; c < C; ++c, base += sC, gi += cC, go += P) {
      const T gO = *go;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (ok[k]) {
          atomic_add(gi + coff[k], w[k] * gO);
          const T v = __ldg(base + off[k]);
          gix += v * dx[k] * gO;
          giy += v * dy[k] * gO;
          giz += v * dz[k] * gO;
        }
    }
    T* gg = ggrid + idx * 3;
    gg[0] = ax.mult * (gix * (T)W / (T)2);
    gg[1] = ay.mult * (giy * (T)H / (T)2);
    gg[2] = az.mult * (giz * (T)D / (T)2);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
gs3d_dbwd_kernel(const T* __restrict__ gg_inp, const T* __restrict__ gg_grid,
                 const T* __restrict__ input, long long sN, long long sC, long long sD,
                 long long sH, long long sW, const T* __restrict__ grid,
                 const T* __restrict__ gout, T* __restrict__ ginp, T* __restrict__ ggrid,
                 T* __restrict__ ggout, int N, int C, int D, int H, int W, long long P) {
  const long long total = (long long)N * P;
  const long long cD = (long long)H * W, cC = (long long)D * H * W;
  for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * kThreads) {
    const long long n = idx / P, p = idx - n * P;
    const T* g = grid + idx * 3;
    const Axis<T> ax = make_axis<T>(g[0], W), ay = make_axis<T>(g[1], H),
                  az = make_axis<T>(g[2], D);
    const T qx = gg_grid[idx * 3 + 0], qy = gg_grid[idx * 3 + 1], qz = gg_grid[idx * 3 + 2];
    const T scx = (T)0.5 * (T)W * ax.mult, scy = (T)0.5 * (T)H * ay.mult,
            scz = (T)0.5 * (T)D * az.mult;
    const T sxy = scx * scy, sxz = scx * scz, syz = scy * scz;
    T w[8], dx[8], dy[8], dz[8], tmp[8], mx[8], my[8], mz[8];
    long long off[8], coff[8];
    bool ok[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int bx = k & 1, by = (k >> 1) & 1, bz = k >> 2;
      const T sx = bx ? (T)1 : (T)-1, sy = by ? (T)1 : (T)-1, sz = bz ? (T)1 : (T)-1;
      w[k] = ax.a[bx] * ay.a[by] * az.a[bz];
      dx[k] = sx * ay.a[by] * az.a[bz];
      dy[k] = sy * ax.a[bx] * az.a[bz];
      dz[k] = sz * ax.a[bx] * ay.a[by];
      // tmp_k = sum_axis gg_grid_axis * scale_axis * d w_k / d axis
      tmp[k] = qx * scx * dx[k] + qy * scy * dy[k] + qz * scz * dz[k];
      // mixed second derivatives contracted with gg_grid
      const T dxy = sx * sy * az.a[bz], dxz = sx * sz * ay.a[by], dyz = sy * sz * ax.a[bx];
      mx[k] = qy * dxy * sxy + qz * dxz * sxz;
      my[k] = qx * dxy * sxy + qz * dyz * syz;
      mz[k] = qx * dxz * sxz + qy * dyz * syz;
      ok[k] = (bx ? ax.in1 : ax.in0) && (by ? ay.in1 : ay.in0) && (bz ? az.in1 : az.in0);
      off[k] = (long long)(az.i0 + bz) * sD + (long long)(ay.i0 + by) * sH +
               (long long)(ax.i0 + bx) * sW;
      coff[k] = (long long)(az.i0 + bz) * cD + (long long)(ay.i0 + by) * W + (ax.i0 + bx);
    }
    const T* base = input + n * sN;
    const T* ggi = gg_inp + n * (long long)C * cC;
    T* gi = ginp + n * (long long)C * cC;
    const T* go = gout + n * (long long)C * P + p;
    T* ggo = ggout + n * (long long)C * P + p;
    T gix = (T)0, giy = (T)0, giz = (T)0;
    for (int c = 0; c < C; ++c, base += sC, ggi += cC, gi += cC, go += P, ggo += P) {
      const T gO = *go;
      T acc = (T)0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (ok[k]) {
          atomic_add(gi + coff[k], tmp[k] * gO);
          const T q = __ldg(ggi + coff[k]);
          const T v = __ldg(base + off[k]);
          gix += q * dx[k] * gO * scx + v * mx[k] * gO;
          giy += q * dy[k] * gO * scy + v * my[k] * gO;
          giz += q * dz[k] * gO * scz + v * mz[k] * gO;
          acc += q * w[k] + v * tmp[k];
        }
      *ggo = acc;
    }
    T* gg = ggrid + idx * 3;
    gg[0] = gix; gg[1] = giy; gg[2] = giz;
  }
}

template <typename T>
int fwd(const T* input, const int64_t* istr, const T* grid, T* output, int32_t* cidx, int N, int C,
        int D, int H, int W, int64_t P, cudaStream_t s) {
  if (N < 0 || C < 0 || D <= 0 || H <= 0 || W <= 0 || P < 0 || !istr) return SR_EINVAL;
  if ((long long)N * P == 0 || (C == 0 && !cidx)) return SR_OK;
  if (!grid || (C > 0 && (!input || !output))) return SR_EINVAL;
  gs3d_fwd_kernel<T><<<sr_grid_for((long long)N * P, kThreads, 16), kThreads, 0, s>>>(
      input, istr[0], istr[1], istr[2], istr[3], istr[4], grid, output, cidx, N, C, D, H, W, P);
  return sr_launch_status();
}
template <typename T>
int bwd(const T* input, const int64_t* istr, const T* grid, const T* gout, T* ginp, T* ggrid,
        int N, int C, int D, int H, int W, int64_t P, cudaStream_t s) {
  if (N < 0 || C < 0 || D <= 0 || H <= 0 || W <= 0 || P < 0 || !istr) return SR_EINVAL;
  if ((long long)N * P == 0) return SR_OK;
  if (!grid || !ggrid || (C > 0 && (!input || !gout || !ginp))) return SR_EINVAL;
  gs3d_bwd_kernel<T><<<sr_grid_for((long long)N * P, kThreads, 16), kThreads, 0, s>>>(
      input, istr[0], istr[1], istr[2], istr[3], istr[4], grid, gout, ginp, ggrid, N, C, D, H, W,
      P);
  return sr_launch_status();
}
template <typename T>
int dbwd(const T* ggi, const T* ggg, const T* input, const int64_t* istr, const T* grid,
         const T* gout, T* ginp, T* ggrid, T* ggout, int N, int C, int D, int H, int W, int64_t P,
         cudaStream_t s) {
  if (N < 0 || C < 0 || D <= 0 || H <= 0 || W <= 0 || P < 0 || !istr) return SR_EINVAL;
  if ((long long)N * P == 0) return SR_OK;
  if (!ggg || !grid || !ggrid || (C > 0 && (!ggi || !input || !gout || !ginp || !ggout)))
    return SR_EINVAL;
  gs3d_dbwd_kernel<T><<<sr_grid_for((long long)N * P, kThreads, 16), kThreads, 0, s>>>(
      ggi, ggg, input, istr[0], istr[1], istr[2], istr[3], istr[4], grid, gout, ginp, ggrid, ggout,
      N, C, D, H, W, P);
  return sr_launch_status();
}

}  // namespace

extern "C" {
int sr_grid_sample3d_fwd_f32(const float* input, const int64_t* istr, const float* grid,
                             float* output, int32_t* corner_idx, int N, int C, int D, int H, int W,
                             int64_t P, cudaStream_t s) {
  return fwd<float>(input, istr, grid, output, corner_idx, N, C, D, H, W, P, s);
}
int sr_grid_sample3d_bwd_f32(const float* input, const int64_t* istr, const float* grid,
                             const float* grad_output, float* grad_input, float* grad_grid, int N,
                             int C, int D, int H, int W, int64_t P, cudaStream_t s) {
  return bwd<float>(input, istr, grid, grad_output, grad_input, grad_grid, N, C, D, H, W, P, s);
}
int sr_grid_sample3d_dbwd_f32(const float* gg_input, const float* gg_grid, const float* input,
                              const int64_t* istr, const float* grid, const float* grad_output,
                              float* grad_input, float* grad_grid, float* grad_grad_output, int N,
                              int C, int D, int H, int W, int64_t P, cudaStream_t s) {
  return dbwd<float>(gg_input, gg_grid, input, istr, grid, grad_output, grad_input, grad_grid,
                     grad_grad_output, N, C, D, H, W, P, s);
}
int sr_grid_sample3d_fwd_f64(const double* input, const int64_t* istr, const double* grid,
                             double* output, int32_t* corner_idx, int N, int C, int D, int H,
                             int W, int64_t P, cudaStream_t s) {
  return fwd<double>(input, istr, grid, output, corner_idx, N, C, D, H, W, P, s);
}
int sr_grid_sample3d_bwd_f64(const double* input, const int64_t* istr, const double* grid,
                             const double* grad_output, double* grad_input, double* grad_grid,
                             int N, int C, int D, int H, int W, int64_t P, cudaStream_t s) {
  return bwd<double>(input, istr, grid, grad_output, grad_input, grad_grid, N, C, D, H, W, P, s);
}
int sr_grid_sample3d_dbwd_f64(const double* gg_input, const double* gg_grid, const double* input,
                              const int64_t* istr, const double* grid, const double* grad_output,
                              double* grad_input, double* grad_grid, double* grad_grad_output,
                              int N, int C, int D, int H, int W, int64_t P, cudaStream_t s) {
  return dbwd<double>(gg_input, gg_grid, input, istr, grid, grad_output, grad_input, grad_grid,
                      grad_grad_output, N, C, D, H, W, P, s);
}
}
