// (2n-1) trilinear upsample + "is boundary" flag, and its adjoint (SURVEY.md rows a21 / K10-K13).
//
// Semantics follow MCAcc/cuda/interp2x_boundary3d_kernel.cu:10-239 (3-D) and
// interp2x_boundary2d_kernel.cu:11-140 (2-D) of the reference: an output voxel whose
// coordinates are all even copies its source; otherwise it is the mean of the 2 / 4 / 8
// sources that surround it (summed left to right in the reference's tap order, then divided
// by a power of two) and is a boundary voxel iff those sources disagree on `v > balance`.
//
// HBM-bound: 5 B written per output voxel, sources come from L1/L2.  One thread per output
// voxel along x (coalesced 4 B + 1 B stores), grid = multiple of the SM count, grid-stride.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

// taps[] order reproduces the reference: it depends on which axes are odd.
//   odd {x}        : x-,x+            odd {y}: y-,y+          odd {z}: z-,z+
//   odd {x,y} (z even): (y-,x-),(y-,x+),(y+,x-),(y+,x+)            -> x fastest
//   odd {y,z} (x even): (z-,y-),(z+,y-),(z-,y+),(z+,y+)            -> z fastest
//   odd {x,z} (y even): (z-,x-),(z+,x-),(z-,x+),(z+,x+)            -> z fastest
//   odd {x,y,z}        : x fastest, then y, then z
// One CTA per output row (b, z, y): the parities of y and z -- and with them the tap pattern -- are
// uniform in the CTA, and thread t produces the output pair x = 2t (even) and x = 2t+1 (odd) from the
// source columns t and t+1 of the (up to four) source rows, so there is no per-voxel div/mod and no
// divergent switch (the first version had both and ran at 0.4 TB/s).
__global__ void __launch_bounds__(kThreads)
interp2x3d_fwd_kernel(const float* __restrict__ in, float* __restrict__ out,
                      uint8_t* __restrict__ bnd, int bc, int d, int h, int w, float balance) {
  const int od = 2 * d - 1, oh = 2 * h - 1, ow = 2 * w - 1;
  const long long rows = (long long)bc * od * oh;
  for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
    const int y = (int)(row % oh);
    const int z = (int)((row / oh) % od);
    const long long b = row / ((long long)oh * od);
    const int oy = y & 1, oz = z & 1;
    const int y0 = (y - oy) >> 1, y1 = (y + oy) >> 1, z0 = (z - oz) >> 1, z1 = (z + oz) >> 1;
    const float* s00 = in + ((b * d + z0) * (long long)h + y0) * w;   // (z0, y0)
    const float* s01 = in + ((b * d + z0) * (long long)h + y1) * w;   // (z0, y1)
    const float* s10 = in + ((b * d + z1) * (long long)h + y0) * w;   // (z1, y0)
    const float* s11 = in + ((b * d + z1) * (long long)h + y1) * w;   // (z1, y1)
    float* orow = out + row * ow;
    uint8_t* brow = bnd + row * ow;
    for (int t = threadIdx.x; t < w; t += kThreads) {
      const bool has_odd = t + 1 < w;
      const int t1 = has_odd ? t + 1 : t;
      // a[z][y][x]
      const float a000 = __ldg(s00 + t), a001 = __ldg(s00 + t1);
      const float a010 = oy ? __ldg(s01 + t) : a000, a011 = oy ? __ldg(s01 + t1) : a001;
      const float a100 = oz ? __ldg(s10 + t) : a000, a101 = oz ? __ldg(s10 + t1) : a001;
      const float a110 = (oy & oz) ? __ldg(s11 + t) : (oz ? a100 : a010);
      const float a111 = (oy & oz) ? __ldg(s11 + t1) : (oz ? a101 : a011);
      float ve, vo;      // even-x and odd-x outputs
      bool de, dodd;     // their boundary flags
      const bool f0 = a000 > balance;
      // sums in the reference's tap order (see the table above); /2 /4 /8 are exact
      if (!oy && !oz) {
        ve = a000; de = false;
        vo = __fadd_rn(a000, a001) * 0.5f; dodd = (a001 > balance) != f0;
      } else if (oy && !oz) {
        ve = __fadd_rn(a000, a010) * 0.5f; de = (a010 > balance) != f0;
        vo = __fadd_rn(__fadd_rn(__fadd_rn(a000, a001), a010), a011) * 0.25f;
        dodd = ((a001 > balance) != f0) | ((a010 > balance) != f0) | ((a011 > balance) != f0);
      } else if (!oy && oz) {
        ve = __fadd_rn(a000, a100) * 0.5f; de = (a100 > balance) != f0;
        vo = __fadd_rn(__fadd_rn(__fadd_rn(a000, a100), a001), a101) * 0.25f;     // z fastest
        dodd = ((a100 > balance) != f0) | ((a001 > balance) != f0) | ((a101 > balance) != f0);
      } else {
        ve = __fadd_rn(__fadd_rn(__fadd_rn(a000, a100), a010), a110) * 0.25f;     // z fastest
        de = ((a100 > balance) != f0) | ((a010 > balance) != f0) | ((a110 > balance) != f0);
        vo = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(a000, a001), a010), a011), a100),
                                           a101), a110), a111) * 0.125f;           // x, then y, then z
        dodd = ((a001 > balance) != f0) | ((a010 > balance) != f0) | ((a011 > balance) != f0) |
               ((a100 > balance) != f0) | ((a101 > balance) != f0) | ((a110 > balance) != f0) |
               ((a111 > balance) != f0);
      }
      orow[2 * t] = ve;
      brow[2 * t] = de ? 1 : 0;
      if (has_odd) {
        orow[2 * t + 1] = vo;
        brow[2 * t + 1] = dodd ? 1 : 0;
      }
    }
  }
}

// adjoint: one thread per input voxel, 27 taps in the reference's order
// (centre, 6 edge taps, 12 face taps xy/xz/yz, 8 corner taps).
__global__ void __launch_bounds__(kThreads)
interp2x3d_bwd_kernel(const float* __restrict__ gout, float* __restrict__ gin, int bc, int d,
                      int h, int w) {
  const int od = 2 * d - 1, oh = 2 * h - 1, ow = 2 * w - 1;
  const long long per = (long long)d * h * w;
  const long long total = per * bc;
  for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * kThreads) {
    const int x = (int)(idx % w);
    const int y = (int)((idx / w) % h);
    const int z = (int)((idx / ((long long)w * h)) % d);
    const long long b = idx / per;
    const float* g = gout + b * (long long)od * oh * ow;
    const bool xm = x > 0, xp = x < w - 1, ym = y > 0, yp = y < h - 1, zm = z > 0, zp = z < d - 1;
#define G(dz, dy, dx) __ldg(g + ((long long)(2 * z + (dz)) * oh + (2 * y + (dy))) * ow + (2 * x + (dx)))
    float acc = G(0, 0, 0);
    if (xm) acc += G(0, 0, -1) * 0.5f;
    if (xp) acc += G(0, 0, 1) * 0.5f;
    if (ym) acc += G(0, -1, 0) * 0.5f;
    if (yp) acc += G(0, 1, 0) * 0.5f;
    if (zm) acc += G(-1, 0, 0) * 0.5f;
    if (zp) acc += G(1, 0, 0) * 0.5f;
    if (xm && ym) acc += G(0, -1, -1) * 0.25f;
    if (xp && ym) acc += G(0, -1, 1) * 0.25f;
    if (xm && yp) acc += G(0, 1, -1) * 0.25f;
    if (xp && yp) acc += G(0, 1, 1) * 0.25f;
    if (xm && zm) acc += G(-1, 0, -1) * 0.25f;
    if (xp && zm) acc += G(-1, 0, 1) * 0.25f;
    if (xm && zp) acc += G(1, 0, -1) * 0.25f;
    if (xp && zp) acc += G(1, 0, 1) * 0.25f;
    if (ym && zm) acc += G(-1, -1, 0) * 0.25f;
    if (yp && zm) acc += G(-1, 1, 0) * 0.25f;
    if (ym && zp) acc += G(1, -1, 0) * 0.25f;
    if (yp && zp) acc += G(1, 1, 0) * 0.25f;
    if (xm && ym && zm) acc += G(-1, -1, -1) * 0.125f;
    if (xp && ym && zm) acc += G(-1, -1, 1) * 0.125f;
    if (xm && yp && zm) acc += G(-1, 1, -1) * 0.125f;
    if (xp && yp && zm) acc += G(-1, 1, 1) * 0.125f;
    if (xm && ym && zp) acc += G(1, -1, -1) * 0.125f;
    if (xp && ym && zp) acc += G(1, -1, 1) * 0.125f;
    if (xm && yp && zp) acc += G(1, 1, -1) * 0.125f;
    if (xp && yp && zp) acc += G(1, 1, 1) * 0.125f;
#undef G
    gin[idx] = acc;
  }
}

__global__ void __launch_bounds__(kThreads)
interp2x2d_fwd_kernel(const float* __restrict__ in, float* __restrict__ out,
                      uint8_t* __restrict__ bnd, int bc, int h, int w, float balance) {
  const int oh = 2 * h - 1, ow = 2 * w - 1;
  const long long per = (long long)oh * ow, total = per * bc;
  for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * kThreads) {
    const int x = (int)(idx % ow), y = (int)((idx / ow) % oh);
    const long long b = idx / per;
    const float* src = in + b * (long long)h * w;
    const int ox = x & 1, oy = y & 1;
    const int x0 = (x - ox) >> 1, x1 = (x + ox) >> 1, y0 = (y - oy) >> 1, y1 = (y + oy) >> 1;
    float v[4];
    int n;
    if (!ox && !oy) { v[0] = src[(long long)y0 * w + x0]; n = 1; }
    else if (!ox) { v[0] = src[(long long)y0 * w + x0]; v[1] = src[(long long)y1 * w + x0]; n = 2; }
    else if (!oy) { v[0] = src[(long long)y0 * w + x0]; v[1] = src[(long long)y0 * w + x1]; n = 2; }
    else {
      v[0] = src[(long long)y0 * w + x0]; v[1] = src[(long long)y0 * w + x1];
      v[2] = src[(long long)y1 * w + x0]; v[3] = src[(long long)y1 * w + x1]; n = 4;
    }
    float sum = v[0];
    const bool f0 = v[0] > balance;
    bool differ = false;
    for (int t = 1; t < n; ++t) { sum = __fadd_rn(sum, v[t]); differ |= ((v[t] > balance) != f0); }
    out[idx] = sum * (n == 1 ? 1.0f : (n == 2 ? 0.5f : 0.25f));
    bnd[idx] = differ ? 1 : 0;
  }
}

__global__ void __launch_bounds__(kThreads)
interp2x2d_bwd_kernel(const float* __restrict__ gout, float* __restrict__ gin, int bc, int h,
                      int w) {
  const int oh = 2 * h - 1, ow = 2 * w - 1;
  const long long per = (long long)h * w, total = per * bc;
  for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * kThreads) {
    const int x = (int)(idx % w), y = (int)((idx / w) % h);
    const long long b = idx / per;
    const float* g = gout + b * (long long)oh * ow;
    const bool xm = x > 0, xp = x < w - 1, ym = y > 0, yp = y < h - 1;
#define G(dy, dx) g[(long long)(2 * y + (dy)) * ow + (2 * x + (dx))]
    float acc = G(0, 0);
    if (xm) acc += G(0, -1) * 0.5f;
    if (xp) acc += G(0, 1) * 0.5f;
    if (ym) acc += G(-1, 0) * 0.5f;
    if (yp) acc += G(1, 0) * 0.5f;
    if (xm && ym) acc += G(-1, -1) * 0.25f;
    if (xp && ym) acc += G(-1, 1) * 0.25f;
    if (xm && yp) acc += G(1, -1) * 0.25f;
    if (xp && yp) acc += G(1, 1) * 0.25f;
#undef G
    gin[idx] = acc;
  }
}

}  // namespace

extern "C" {
int sr_interp2x3d_fwd_f32(const float* in, float* out, uint8_t* is_boundary, int bc, int d, int h,
                          int w, float balance, cudaStream_t s) {
  if (bc <= 0 || d <= 0 || h <= 0 || w <= 0 || !in || !out || !is_boundary) return SR_EINVAL;
  long long total = (long long)bc * (2 * d - 1) * (2 * h - 1) * (2 * w - 1);
  interp2x3d_fwd_kernel<<<sr_grid_for(total, kThreads, 16), kThreads, 0, s>>>(in, out, is_boundary,
                                                                              bc, d, h, w, balance);
  return sr_launch_status();
}
int sr_interp2x3d_bwd_f32(const float* grad_out, float* grad_in, int bc, int d, int h, int w,
                          cudaStream_t s) {
  if (bc <= 0 || d <= 0 || h <= 0 || w <= 0 || !grad_out || !grad_in) return SR_EINVAL;
  long long total = (long long)bc * d * h * w;
  interp2x3d_bwd_kernel<<<sr_grid_for(total, kThreads, 16), kThreads, 0, s>>>(grad_out, grad_in, bc,
                                                                              d, h, w);
  return sr_launch_status();
}
int sr_interp2x2d_fwd_f32(const float* in, float* out, uint8_t* is_boundary, int bc, int h, int w,
                          float balance, cudaStream_t s) {
  if (bc <= 0 || h <= 0 || w <= 0 || !in || !out || !is_boundary) return SR_EINVAL;
  long long total = (long long)bc * (2 * h - 1) * (2 * w - 1);
  interp2x2d_fwd_kernel<<<sr_grid_for(total, kThreads, 16), kThreads, 0, s>>>(in, out, is_boundary,
                                                                              bc, h, w, balance);
  return sr_launch_status();
}
int sr_interp2x2d_bwd_f32(const float* grad_out, float* grad_in, int bc, int h, int w,
                          cudaStream_t s) {
  if (bc <= 0 || h <= 0 || w <= 0 || !grad_out || !grad_in) return SR_EINVAL;
  long long total = (long long)bc * h * w;
  interp2x2d_bwd_kernel<<<sr_grid_for(total, kThreads, 16), kThreads, 0, s>>>(grad_out, grad_in, bc,
                                                                              h, w);
  return sr_launch_status();
}
}
