// Front-normal network of the normal-map step (generate_normals.py:116-166 of the reference: PIFuHD's netF, pix2pixHD's
// GlobalGenerator(3, 3, 64, 4 downsamplings, 9 blocks, instance norm), then the map back onto the frame).
//
// Every convolution is an implicit-im2col pack into the tiled split-bf16 operand layout of the tensor-core layer
// kernel (tc_gemm.cu, the layout sr_tc_pack_rows writes) followed by sr_tc_linear: activations are fp32 channels-last
// [B,H,W,C], GEMM row m = (b*Ho + oy)*Wo + ox, column k = (ky*kw + kx)*Cin + ci (tap-major, channel-minor, the order
// the loader reorders the weights to).  This file holds the glue around that GEMM:
//   * conv_pack_kernel: rows [row0, row0+rows) of the im2col matrix, zero or reflection padding, stride 1 or 2, and
//     the gather form of ConvTranspose2d (iy = (oy + p - ky) / s when that divides exactly and lies in range);
//   * instance-norm statistics: per (sample, channel) sums in float64 over fixed 512-pixel slices, then a fixed-order
//     sum of the slices -- no atomics, and a sample's order does not depend on the batch size;
//   * instance-norm apply: (y - mean) * rstd, optional ReLU, optional residual add;
//   * normal_unwarp_kernel: grid_sample of the net output back onto the frame and the 8-bit quantisation of
//     generate_normals.py:149-165, one correctly rounded fp32 operation at a time (nvcc contracts none of them) in the
//     order of torch's CPU grid sampler and of the script's numpy expressions.
#include "tc_common.cuh"

namespace sr_nn {
using namespace sr_tc;

constexpr int kThreads = 256;
constexpr int kSlice = 512;   // pixels per partial sum of the instance-norm statistics

struct ConvGeom {
  const float* x;
  int H, W, Cin;       // input [B,H,W,Cin]
  int Ho, Wo;          // output size
  int kh, kw, stride, pad;
  int reflect;         // 1: reflection padding, 0: zero padding
  int transposed;      // 1: ConvTranspose2d in gather form
  int K, KC;           // K = kh*kw*Cin, KC = ceil(K / 32) chunks
  long long row0, rows, MT;
};

__device__ __forceinline__ int reflect_idx(int i, int n) {   // ReflectionPad2d: -1 -> 1, n -> n - 2 (pad < n)
  i = i < 0 ? -i : i;
  return i >= n ? 2 * n - 2 - i : i;
}

// input pixel (b, iy, ix) a tap (ky, kx) of output (oy, ox) reads, as a flat pixel index; -1 = a zero
__device__ __forceinline__ long long src_pixel(const ConvGeom& g, int b, int oy, int ox, int ky, int kx) {
  int iy, ix;
  if (g.transposed) {
    const int ty = oy + g.pad - ky, tx = ox + g.pad - kx;
    if (ty < 0 || tx < 0 || ty % g.stride != 0 || tx % g.stride != 0) return -1;
    iy = ty / g.stride;
    ix = tx / g.stride;
    if (iy >= g.H || ix >= g.W) return -1;
  } else {
    iy = oy * g.stride - g.pad + ky;
    ix = ox * g.stride - g.pad + kx;
    if (g.reflect) {
      iy = reflect_idx(iy, g.H);
      ix = reflect_idx(ix, g.W);
    } else if (iy < 0 || iy >= g.H || ix < 0 || ix >= g.W) {
      return -1;
    }
  }
  return ((long long)b * g.H + iy) * g.W + ix;
}

// One thread per (row, group of 8 columns), ordered as pack_rows_kernel: the 16 B stores of a warp are contiguous.
// kVec (Cin % 8 == 0): a group lies inside one tap and is two 16 B loads.
template <bool kVec>
__global__ void __launch_bounds__(kThreads) conv_pack_kernel(const __grid_constant__ ConvGeom g,
                                                             __nv_bfloat16* __restrict__ dst) {
  const long long total = g.MT * BM * (long long)g.KC * 4;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(idx % BM);
    const long long rest = idx / BM;
    const int grp = (int)(rest % (g.KC * 4));
    const long long mt = rest / (g.KC * 4);
    const long long lrow = mt * BM + r;
    const int k0 = grp * 8;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
    if (lrow < g.rows && k0 < g.K) {
      const long long m = g.row0 + lrow;
      const int ox = (int)(m % g.Wo);
      const long long t = m / g.Wo;
      const int oy = (int)(t % g.Ho);
      const int b = (int)(t / g.Ho);
      if constexpr (kVec) {
        const int tap = k0 / g.Cin, c0 = k0 - tap * g.Cin;
        const long long p = src_pixel(g, b, oy, ox, tap / g.kw, tap % g.kw);
        if (p >= 0) {
          const float4* s4 = reinterpret_cast<const float4*>(g.x + p * g.Cin + c0);
          const float4 a = __ldg(s4), c = __ldg(s4 + 1);
          v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
          v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int k = k0 + e;
          if (k < g.K) {
            const int tap = k / g.Cin, ci = k - tap * g.Cin;
            const long long p = src_pixel(g, b, oy, ox, tap / g.kw, tap % g.kw);
            if (p >= 0) v[e] = __ldg(g.x + p * g.Cin + ci);
          }
        }
      }
    }
    __align__(16) __nv_bfloat16 p1[8], p2[8], p3[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) split3(v[e], p1[e], p2[e], p3[e]);
    const int kc = grp >> 2, k8 = grp & 3;
    const size_t off = (size_t)k8 * (BM * 8) + (size_t)(r >> 3) * 64 + (r & 7) * 8;
    *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, g.KC, 0) + off) = *reinterpret_cast<uint4*>(p1);
    *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, g.KC, 1) + off) = *reinterpret_cast<uint4*>(p2);
    if constexpr (kPlanes == 3)
      *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, g.KC, kPlanes - 1) + off) = *reinterpret_cast<uint4*>(p3);
  }
}

// Block (32 channels x 8 pixel lanes) of slice s of sample b: float64 sum and sum of squares of 512 pixels, the 8
// lanes added in lane order.  partial [B][S][C][2].
__global__ void __launch_bounds__(kThreads) in_partial_kernel(const float* __restrict__ y, long long HW, int C, int S,
                                                              double* __restrict__ partial) {
  __shared__ double sh[8][32][2];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int s = blockIdx.x, c = blockIdx.y * 32 + tx, b = blockIdx.z;
  const long long p0 = (long long)s * kSlice, p1 = min(HW, p0 + kSlice);
  double s1 = 0.0, s2 = 0.0;
  if (c < C) {
    const float* yb = y + (size_t)b * HW * C + c;
    for (long long p = p0 + ty; p < p1; p += 8) {
      const double v = (double)__ldg(yb + (size_t)p * C);
      s1 += v;
      s2 += v * v;
    }
  }
  sh[ty][tx][0] = s1;
  sh[ty][tx][1] = s2;
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int j = 1; j < 8; ++j) {
      s1 += sh[j][tx][0];
      s2 += sh[j][tx][1];
    }
    double* o = partial + (((size_t)b * S + s) * C + c) * 2;
    o[0] = s1;
    o[1] = s2;
  }
}

// One thread per (sample, channel): the slices in order -> mean and 1 / sqrt(biased var + eps)
__global__ void in_finish_kernel(const double* __restrict__ partial, int B, long long HW, int C, int S,
                                 float* __restrict__ mean, float* __restrict__ rstd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  double s1 = 0.0, s2 = 0.0;
  for (int s = 0; s < S; ++s) {
    const double* p = partial + (((size_t)b * S + s) * C + c) * 2;
    s1 += p[0];
    s2 += p[1];
  }
  const double mu = s1 / (double)HW;
  const double var = fmax(s2 / (double)HW - mu * mu, 0.0);
  mean[i] = (float)mu;
  rstd[i] = (float)(1.0 / sqrt(var + 1e-5));
}

// out = relu?((y - mean) * rstd) (+ residual); kVec: 4 channels per thread (C % 4 == 0)
template <bool kVec>
__global__ void __launch_bounds__(kThreads) in_apply_kernel(const float* y, long long HW, int C, long long n,
                                                            const float* __restrict__ mean,
                                                            const float* __restrict__ rstd, const float* residual,
                                                            int relu, float* out) {
  constexpr int V = kVec ? 4 : 1;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n / V;
       q += (long long)gridDim.x * blockDim.x) {
    const long long i = q * V;
    const int c = (int)(i % C);
    const long long bc = (i / ((long long)HW * C)) * C + c;
    float v[V], r[V];
    if constexpr (kVec) {
      const float4 a = *reinterpret_cast<const float4*>(y + i);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
      if (residual) {
        const float4 rr = *reinterpret_cast<const float4*>(residual + i);
        r[0] = rr.x; r[1] = rr.y; r[2] = rr.z; r[3] = rr.w;
      }
    } else {
      v[0] = y[i];
      if (residual) r[0] = residual[i];
    }
#pragma unroll
    for (int j = 0; j < V; ++j) {
      float t = (v[j] - mean[bc + j]) * rstd[bc + j];
      if (relu) t = fmaxf(t, 0.f);
      v[j] = residual ? t + r[j] : t;
    }
    if constexpr (kVec)
      *reinterpret_cast<float4*>(out + i) = make_float4(v[0], v[1], v[2], v[3]);
    else
      out[i] = v[0];
  }
}

// grid_sample(net, coords, bilinear, zeros, align_corners=True) at pixel (r, c) of frame b, then
// generate_normals.py:155-165.  The float32 order is torch's CPU path: coords = 2*(c - x)/w - 1 (true division),
// ix = (g + 1) * ((S - 1) / 2), corner weights from floor(ix), the four corners added nw, ne, sw, se; then numpy's
// (n * 0.5 + 0.5)[::-1] * 255 and astype(uint8) (truncation).
__global__ void __launch_bounds__(kThreads) normal_unwarp_kernel(const float* __restrict__ net, int B, int S,
                                                                 const float* __restrict__ boxes,
                                                                 const uint8_t* __restrict__ fg, int H, int W,
                                                                 uint8_t* __restrict__ out) {
  const long long HW = (long long)H * W, n = (long long)B * HW;
  const float scale = __fdiv_rn((float)(S - 1), 2.f);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / HW);
    const long long pix = i - (long long)b * HW;
    const int r = (int)(pix / W), c = (int)(pix - (long long)r * W);
    const float bx = boxes[4 * b], by = boxes[4 * b + 1], bw = boxes[4 * b + 2], bh = boxes[4 * b + 3];
    const float gx = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fsub_rn((float)c, bx)), bw), 1.f);
    const float gy = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fsub_rn((float)r, by)), bh), 1.f);
    const float ix = __fmul_rn(__fadd_rn(gx, 1.f), scale), iy = __fmul_rn(__fadd_rn(gy, 1.f), scale);
    const float x_w = floorf(ix), y_n = floorf(iy);
    const float we = __fsub_rn(ix, x_w), e = __fsub_rn(1.f, we);
    const float wn = __fsub_rn(iy, y_n), ws = __fsub_rn(1.f, wn);
    const float w_nw = __fmul_rn(ws, e), w_ne = __fmul_rn(ws, we), w_sw = __fmul_rn(wn, e), w_se = __fmul_rn(wn, we);
    const int x0 = (int)x_w, y0 = (int)y_n;
    const bool in_w = x0 >= 0 && x0 < S, in_e = x0 + 1 >= 0 && x0 + 1 < S;
    const bool in_n = y0 >= 0 && y0 < S, in_s = y0 + 1 >= 0 && y0 + 1 < S;
    const float* base = net + (size_t)b * S * S * 3;
    float v[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float nw = in_n && in_w ? base[((size_t)y0 * S + x0) * 3 + ch] : 0.f;
      const float ne = in_n && in_e ? base[((size_t)y0 * S + x0 + 1) * 3 + ch] : 0.f;
      const float sw = in_s && in_w ? base[((size_t)(y0 + 1) * S + x0) * 3 + ch] : 0.f;
      const float se = in_s && in_e ? base[((size_t)(y0 + 1) * S + x0 + 1) * 3 + ch] : 0.f;
      float a = __fadd_rn(__fmul_rn(nw, w_nw), __fmul_rn(ne, w_ne));
      a = __fadd_rn(a, __fmul_rn(sw, w_sw));
      v[ch] = __fadd_rn(a, __fmul_rn(se, w_se));
    }
    float sq = __fmul_rn(v[0], v[0]);
    sq = __fadd_rn(sq, __fmul_rn(v[1], v[1]));
    sq = __fadd_rn(sq, __fmul_rn(v[2], v[2]));
    const bool zero = __fsqrt_rn(sq) < 1e-4f || (fg != nullptr && fg[i] == 0);
    uint8_t* o = out + i * 3;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const float q = __fmul_rn(__fadd_rn(__fmul_rn(v[2 - j], 0.5f), 0.5f), 255.f);
      const int t = zero ? 0 : (int)q;
      o[j] = (uint8_t)(t < 0 ? 0 : (t > 255 ? 255 : t));
    }
  }
}

}  // namespace sr_nn

int sr_conv_pack(const float* x, int B, int H, int W, int Cin, int kh, int kw, int stride, int pad, int reflect,
                 int transposed, int Ho, int Wo, int64_t row0, int64_t rows, void* dst, cudaStream_t s) {
  using namespace sr_nn;
  if (!x || !dst || B <= 0 || H <= 0 || W <= 0 || Cin <= 0 || kh <= 0 || kw <= 0 || Ho <= 0 || Wo <= 0) return SR_EINVAL;
  if ((stride != 1 && stride != 2) || pad < 0 || (reflect && (transposed || pad >= H || pad >= W))) return SR_EINVAL;
  if (row0 < 0 || rows <= 0 || row0 + rows > (int64_t)B * Ho * Wo) return SR_EINVAL;
  ConvGeom g;
  g.x = x; g.H = H; g.W = W; g.Cin = Cin; g.Ho = Ho; g.Wo = Wo; g.kh = kh; g.kw = kw; g.stride = stride; g.pad = pad;
  g.reflect = reflect; g.transposed = transposed; g.K = kh * kw * Cin; g.KC = (g.K + 31) / 32;
  g.row0 = row0; g.rows = rows; g.MT = (rows + BM - 1) / BM;
  const long long total = g.MT * BM * (long long)g.KC * 4;
  if (Cin % 8 == 0)
    conv_pack_kernel<true><<<sr_grid_for(total, kThreads, 8), kThreads, 0, s>>>(g, (__nv_bfloat16*)dst);
  else
    conv_pack_kernel<false><<<sr_grid_for(total, kThreads, 8), kThreads, 0, s>>>(g, (__nv_bfloat16*)dst);
  return sr_launch_status();
}

int64_t sr_instance_norm_partial_bytes(int B, int64_t HW, int C) {
  const int64_t S = (HW + sr_nn::kSlice - 1) / sr_nn::kSlice;
  return (int64_t)B * S * C * 2 * (int64_t)sizeof(double);
}

int sr_instance_norm_stats(const float* y, int B, int64_t HW, int C, void* partial, float* mean, float* rstd,
                           cudaStream_t s) {
  using namespace sr_nn;
  if (!y || !partial || !mean || !rstd || B <= 0 || B > 65535 || HW <= 0 || C <= 0) return SR_EINVAL;
  const int64_t S = (HW + kSlice - 1) / kSlice;
  if (S > 0x7fffffff || (C + 31) / 32 > 65535) return SR_EINVAL;
  in_partial_kernel<<<dim3((unsigned)S, (C + 31) / 32, B), kThreads, 0, s>>>(y, HW, C, (int)S, (double*)partial);
  const int rc = sr_launch_status();
  if (rc) return rc;
  in_finish_kernel<<<sr_div_up((long long)B * C, 128), 128, 0, s>>>((const double*)partial, B, HW, C, (int)S, mean,
                                                                    rstd);
  return sr_launch_status();
}

int sr_instance_norm_apply(const float* y, int B, int64_t HW, int C, const float* mean, const float* rstd,
                           const float* residual, int relu, float* out, cudaStream_t s) {
  using namespace sr_nn;
  if (!y || !mean || !rstd || !out || B <= 0 || HW <= 0 || C <= 0) return SR_EINVAL;
  const long long n = (long long)B * HW * C;
  const bool vec = C % 4 == 0 && ((uintptr_t)y | (uintptr_t)out | (uintptr_t)residual) % 16 == 0;
  if (vec)
    in_apply_kernel<true><<<sr_grid_for(n / 4, kThreads, 8), kThreads, 0, s>>>(y, HW, C, n, mean, rstd, residual,
                                                                               relu, out);
  else
    in_apply_kernel<false><<<sr_grid_for(n, kThreads, 8), kThreads, 0, s>>>(y, HW, C, n, mean, rstd, residual, relu,
                                                                            out);
  return sr_launch_status();
}

int sr_normal_unwarp(const float* net, int B, int S, const float* boxes, const uint8_t* fg, int H, int W,
                     uint8_t* out, cudaStream_t s) {
  using namespace sr_nn;
  if (!net || !boxes || !out || B <= 0 || S < 2 || H <= 0 || W <= 0) return SR_EINVAL;
  const long long n = (long long)B * H * W;
  normal_unwarp_kernel<<<sr_grid_for(n, kThreads, 8), kThreads, 0, s>>>(net, B, S, boxes, fg, H, W, out);
  return sr_launch_status();
}
