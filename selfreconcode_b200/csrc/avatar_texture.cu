// Textured rendering of the reconstructed avatar (selfreconcode_b200.avatar): a coverage-weighted mip pyramid of the
// baked atlas and an unlit, trilinear-filtered texture lookup on the fragments of the built-in rasteriser
// (csrc/raster.cu).
//
// sr_texture_mips: the atlas [Ht,Wt,3] uint8 (its own channel order) and a level-0 coverage mask [Ht,Wt] -> every
// level in one float4 buffer, (r, g, b, w) per texel, level after level, row-major.  Level 0 is (c / 255, w = 1 where
// the mask is nonzero, else 0).  W_{l+1} = ceil(W_l / 2), H_{l+1} = ceil(H_l / 2), down to 1x1.  A child texel reduces
// the (up to) 2x2 parents (2i + di, 2j + dj) inside its parent level, in the order (0,0), (0,1), (1,0), (1,1):
//   colour = sum w c / sum w when sum w > 0, else the plain mean of the parents' colours;  w = mean of the parents' w.
// So a chart on a black background keeps its colour at coarse levels instead of fading into the background.  One
// launch per level, one thread per output texel, no atomics: reruns are bit-identical.
//
// sr_shade_textured: one thread per pixel of pix_to_face [N,H,W] (packed n*F + f, -1 = empty) and bary [N,H,W,3]:
//   uv = sum b_i vt[ft[f,i]]; level-l texel coordinates x = u W_l - 0.5, y = (1 - v) H_l - 0.5, bilinear with
//   clamp-to-edge.  Trilinear between levels floor(lambda) and floor(lambda) + 1 by the fraction of
//   lambda = clamp(log2 rho, 0, L - 1), rho = the larger length of d(u Wt, v Ht)/dcol and d(u Wt, v Ht)/drow: the
//   analytic screen-space footprint of the UV map.  With lambda_i the face's affine screen barycentrics at the pixel
//   centre (col j, row i) and Z_i the vertices' depths, b_i = (lambda_i / Z_i) / S, S = sum_j lambda_j / Z_j, so
//   db_i/dx = (lambda_i'/Z_i - b_i S') / S with the constant lambda_i' of the face's edge functions.  The footprint and
//   the texel coordinates run in fp64 (one pixel's uv is a sum of products of fp32 inputs; at a 1680^2 atlas an fp32
//   rounding of uv moves the sample by ~1e-4 texel), the filter weights and the texel blend in fp32.
//   out [N,H,W,4]: (rgb, 1) on covered pixels; (background, 0) elsewhere, with the background a constant colour or
//   the image bg [N,H,W,3] uint8 / 255 (same channel order as the atlas).
//   HBM bound: 8 B face id + 12 B barycentrics read, 16 B written per pixel (+3 B per background pixel with an image);
//   the vertex, face, UV and texel gathers hit L2 (a frame's mesh is a few MB, the texels of neighbouring pixels
//   overlap).
#include "common.cuh"

namespace {

struct Level {
  int w, h;
  long long off;   // first texel of the level in the pyramid
};

__device__ __forceinline__ Level level_of(int W0, int H0, int l) {
  Level v{W0, H0, 0};
  for (int k = 0; k < l; ++k) {
    v.off += (long long)v.w * v.h;
    v.w = (v.w + 1) >> 1;
    v.h = (v.h + 1) >> 1;
  }
  return v;
}

__global__ void __launch_bounds__(256)
mip_level0_kernel(const unsigned char* __restrict__ tex, const unsigned char* __restrict__ cov, long long n,
                  float4* __restrict__ out) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
    out[t] = make_float4(tex[t * 3] / 255.f, tex[t * 3 + 1] / 255.f, tex[t * 3 + 2] / 255.f, cov[t] ? 1.f : 0.f);
}

__global__ void __launch_bounds__(256)
mip_reduce_kernel(const float4* __restrict__ src, int ws, int hs, float4* __restrict__ dst, int wd, int hd) {
  const long long n = (long long)wd * hd;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(t / wd), j = (int)(t % wd);
    float sr = 0.f, sg = 0.f, sb = 0.f, sw = 0.f, pr = 0.f, pg = 0.f, pb = 0.f;
    int cnt = 0;
#pragma unroll
    for (int di = 0; di < 2; ++di) {
#pragma unroll
      for (int dj = 0; dj < 2; ++dj) {
        const int r = 2 * i + di, c = 2 * j + dj;
        if (r >= hs || c >= ws) continue;
        const float4 p = src[(long long)r * ws + c];
        sr += p.w * p.x; sg += p.w * p.y; sb += p.w * p.z; sw += p.w;
        pr += p.x; pg += p.y; pb += p.z;
        ++cnt;
      }
    }
    const float inv = 1.f / (float)cnt;
    dst[t] = sw > 0.f ? make_float4(sr / sw, sg / sw, sb / sw, sw * inv)
                      : make_float4(pr * inv, pg * inv, pb * inv, sw * inv);
  }
}

// bilinear sample of level lv at texel coordinates (x, y), clamp-to-edge
__device__ __forceinline__ float3 bilinear(const float4* __restrict__ mips, const Level& lv, double x, double y) {
  x = fmin(fmax(x, -1.0), (double)lv.w);   // keeps the float -> int conversion defined; clamp-to-edge is unchanged
  y = fmin(fmax(y, -1.0), (double)lv.h);
  const double x0 = floor(x), y0 = floor(y);
  const float fx = (float)(x - x0), fy = (float)(y - y0);
  const int c0 = min(max((int)x0, 0), lv.w - 1), c1 = min(max((int)x0 + 1, 0), lv.w - 1);
  const int r0 = min(max((int)y0, 0), lv.h - 1), r1 = min(max((int)y0 + 1, 0), lv.h - 1);
  const float4* base = mips + lv.off;
  const float4 a = base[(long long)r0 * lv.w + c0], b = base[(long long)r0 * lv.w + c1];
  const float4 c = base[(long long)r1 * lv.w + c0], d = base[(long long)r1 * lv.w + c1];
  const float gx = 1.f - fx, gy = 1.f - fy;
  return make_float3(gy * (gx * a.x + fx * b.x) + fy * (gx * c.x + fx * d.x),
                     gy * (gx * a.y + fx * b.y) + fy * (gx * c.y + fx * d.y),
                     gy * (gx * a.z + fx * b.z) + fy * (gx * c.z + fx * d.z));
}

__global__ void __launch_bounds__(256)
shade_textured_kernel(const long long* __restrict__ pix_to_face, const float* __restrict__ bary, long long N, int H,
                      int W, const float* __restrict__ vs, long long V, const long long* __restrict__ faces,
                      const long long* __restrict__ ft, long long F, const float* __restrict__ vt, long long T,
                      const float4* __restrict__ mips, int Wt, int Ht, int L, const unsigned char* __restrict__ bg,
                      float bg0, float bg1, float bg2, float4* __restrict__ out) {
  const long long total = N * H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long pf = pix_to_face[idx];
    long long vi[3], ti[3];
    bool ok = pf >= 0 && pf < N * F;
    const long long m = ok ? pf / F : 0, f = ok ? pf % F : 0;
    if (ok) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        vi[k] = faces[f * 3 + k];
        ti[k] = ft[f * 3 + k];
        ok = ok && vi[k] >= 0 && vi[k] < V && ti[k] >= 0 && ti[k] < T;
      }
    }
    if (!ok) {
      out[idx] = bg ? make_float4(bg[idx * 3] / 255.f, bg[idx * 3 + 1] / 255.f, bg[idx * 3 + 2] / 255.f, 0.f)
                    : make_float4(bg0, bg1, bg2, 0.f);
      continue;
    }
    const long long pix = idx % ((long long)H * W);
    const double px = (double)(pix % W), py = (double)(pix / W);
    double x[3], y[3], iz[3], u[3], v[3], b[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float* p = vs + (m * V + vi[k]) * 3;
      x[k] = p[0]; y[k] = p[1]; iz[k] = 1.0 / (double)p[2];
      u[k] = vt[ti[k] * 2]; v[k] = vt[ti[k] * 2 + 1];
      b[k] = bary[idx * 3 + k];
    }
    // affine barycentrics at the pixel centre and their constant screen gradients (edge functions / twice the area)
    const double ia = 1.0 / ((x[1] - x[0]) * (y[2] - y[0]) - (x[2] - x[0]) * (y[1] - y[0]));
    const double la[3] = {((x[1] - px) * (y[2] - py) - (x[2] - px) * (y[1] - py)) * ia,
                          ((x[2] - px) * (y[0] - py) - (x[0] - px) * (y[2] - py)) * ia,
                          ((x[0] - px) * (y[1] - py) - (x[1] - px) * (y[0] - py)) * ia};
    const double ldx[3] = {(y[1] - y[2]) * ia, (y[2] - y[0]) * ia, (y[0] - y[1]) * ia};
    const double ldy[3] = {(x[2] - x[1]) * ia, (x[0] - x[2]) * ia, (x[1] - x[0]) * ia};
    double S = 0.0, Sx = 0.0, Sy = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      S += la[k] * iz[k];
      Sx += ldx[k] * iz[k];
      Sy += ldy[k] * iz[k];
    }
    double ux = 0.0, uy = 0.0, vx = 0.0, vy = 0.0, uu = 0.0, vv = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double bk = la[k] * iz[k] / S;
      const double bx = (ldx[k] * iz[k] - bk * Sx) / S, by = (ldy[k] * iz[k] - bk * Sy) / S;
      ux += bx * u[k]; uy += by * u[k]; vx += bx * v[k]; vy += by * v[k];
      uu += b[k] * u[k]; vv += b[k] * v[k];
    }
    const double rho = fmax(sqrt(ux * ux * Wt * Wt + vx * vx * Ht * Ht), sqrt(uy * uy * Wt * Wt + vy * vy * Ht * Ht));
    const double lam = fmin(fmax(log2(rho), 0.0), (double)(L - 1));   // fmax drops a NaN footprint to level 0
    const int l0 = (int)floor(lam);
    const float fr = (float)(lam - l0);
    const Level lv0 = level_of(Wt, Ht, l0);
    float3 c = bilinear(mips, lv0, uu * lv0.w - 0.5, (1.0 - vv) * lv0.h - 0.5);
    if (fr > 0.f) {
      const Level lv1 = level_of(Wt, Ht, min(l0 + 1, L - 1));
      const float3 d = bilinear(mips, lv1, uu * lv1.w - 0.5, (1.0 - vv) * lv1.h - 0.5);
      const float g = 1.f - fr;
      c = make_float3(g * c.x + fr * d.x, g * c.y + fr * d.y, g * c.z + fr * d.z);
    }
    out[idx] = make_float4(c.x, c.y, c.z, 1.f);
  }
}

int levels_of(int Wt, int Ht) {
  int L = 1;
  for (int w = Wt, h = Ht; w > 1 || h > 1; ++L) {
    w = (w + 1) >> 1;
    h = (h + 1) >> 1;
  }
  return L;
}

}  // namespace

extern "C" int sr_texture_mips(const uint8_t* texture, const uint8_t* coverage, int Ht, int Wt, float* mips,
                               cudaStream_t s) {
  if (!texture || !coverage || !mips || Ht <= 0 || Wt <= 0) return SR_EINVAL;
  if (((uintptr_t)mips & 15) != 0) return SR_EINVAL;   // float4 texels
  float4* m = (float4*)mips;
  const long long n0 = (long long)Wt * Ht;
  mip_level0_kernel<<<sr_grid_for(n0, 256, 8), 256, 0, s>>>(texture, coverage, n0, m);
  int rc = sr_launch_status();
  long long off = 0;
  for (int w = Wt, h = Ht; rc == SR_OK && (w > 1 || h > 1);) {
    const int wd = (w + 1) >> 1, hd = (h + 1) >> 1;
    mip_reduce_kernel<<<sr_grid_for((long long)wd * hd, 256, 8), 256, 0, s>>>(m + off, w, h, m + off + (long long)w * h,
                                                                              wd, hd);
    rc = sr_launch_status();
    off += (long long)w * h;
    w = wd;
    h = hd;
  }
  return rc;
}

extern "C" int sr_shade_textured(const int64_t* pix_to_face, const float* bary, int64_t N, int H, int W,
                                 const float* verts_screen, int64_t V, const int64_t* faces, const int64_t* ft,
                                 int64_t F, const float* vt, int64_t T, const float* mips, int Ht, int Wt,
                                 const uint8_t* bg_image, const float* bg_color, float* out, cudaStream_t s) {
  if (!pix_to_face || !bary || !verts_screen || !faces || !ft || !vt || !mips || !out || (!bg_image && !bg_color) ||
      N <= 0 || H <= 0 || W <= 0 || V <= 0 || F <= 0 || T <= 0 || Ht <= 0 || Wt <= 0)
    return SR_EINVAL;
  if ((((uintptr_t)out | (uintptr_t)mips) & 15) != 0) return SR_EINVAL;   // float4 loads and stores
  const float c0 = bg_color ? bg_color[0] : 0.f, c1 = bg_color ? bg_color[1] : 0.f, c2 = bg_color ? bg_color[2] : 0.f;
  shade_textured_kernel<<<sr_grid_for(N * (long long)H * W, 256, 8), 256, 0, s>>>(
      (const long long*)pix_to_face, bary, N, H, W, verts_screen, V, (const long long*)faces, (const long long*)ft, F,
      vt, T, (const float4*)mips, Wt, Ht, levels_of(Wt, Ht), bg_image, c0, c1, c2, (float4*)out);
  return sr_launch_status();
}
