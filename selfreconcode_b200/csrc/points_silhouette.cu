// Soft point-cloud silhouette of the deformed template (model/network.py:495-505): pytorch3d 0.4.0's PointsRasterizer
// (points_per_pixel = K, radius r in NDC units) followed by AlphaCompositor(background_color=None) with all features 1,
// forward and backward, with no pytorch3d.
//
// Input: per frame, the template vertices projected by the camera to (col, row, Z): pixel centres at integer
// (col, row) and Z the view-space depth (raster.screen_vertices, the same projection csrc/raster.cu consumes).
// The rule, in those coordinates (pixel (i, j) = NDC (1-(2j+1)/W, 1-(2i+1)/H), each axis spanning [-1, 1]):
//   d2(p, i, j) = (2/W)^2 (col_p - j)^2 + (2/H)^2 (row_p - i)^2         squared NDC distance
//   p covers (i, j)  iff  Z_p >= 0 and d2 < r^2                          (strict, as CheckPixelInsidePoint)
//   kept(i, j)      = the K covering points with the smallest (Z, index) key
//   w               = 1 - d2 / r^2
//   mask(i, j)      = sum_k w_k prod_{j<k} (1 - w_j) over the kept points in key order  (= 1 - prod_k (1 - w_k))
// The gradient flows through d2 only (the compositor does not read zbuf; the selection is piecewise constant):
//   dmask/dw_p = prod_{q kept, q != p} (1 - w_q),   dw_p/dcol_p = -2 (2/W)^2 (col_p - j) / r^2  (likewise for row).
//
// Kernels (sr_points_silhouette_bin / _forward / _backward):
//  bin      one thread per (frame, rank): the point of that rank in the frame's (Z, index) order (a stable device
//           sort done by the caller) writes one (frame, tile) key per 16x16 pixel tile its disc may touch, into a
//           fixed number of slots per point (sentinel-padded), so the storage is sized on the host without a sync.
//           The caller stable-sorts the keys: every tile's list then stays in (Z, index) order.  16 B written per slot.
//  forward  one CTA per (frame, tile), one thread per pixel: the tile's list streams through shared memory in chunks
//           of 256 points; each pixel accepts covering points in list order until it has K, composites, and keeps
//           O(1) state for the backward: the key of its K-th accepted point (all-ones when it kept fewer than K),
//           the product of its nonzero (1 - w) factors and the number of zero factors (a point within ~r 2^-12 of a
//           pixel centre has w = 1 exactly in fp32, so prod_{q != p} cannot always be formed by division).
//           Per pixel: 20 B written (mask 4, key 8, product 4, zero count 4); per list entry 16 B read by its CTA.
//  backward one thread per (frame, point) walks the pixels of its disc's bounding box in row-major order; it
//           contributes where it covers the pixel and its key is at most the pixel's K-th key, and sums its own
//           screen gradient.  No floating-point atomics: reruns are bit-identical.  Per (point, covered pixel) 20 B
//           read (K-th key 8, product 4, zero count 4, incoming gradient 4; neighbouring points share them in L2);
//           12 B written per point.
// Decisions (coverage, w) use one fixed sequence of correctly rounded fp32 operations in both the forward and the
// backward (ndc_d2 / weight below), so the backward re-takes exactly the forward's decisions.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kTile = SR_POINTS_TILE;   // 16 x 16 pixels per tile, one CTA of 256 pixel threads
constexpr int kChunk = 256;             // list entries staged in shared memory per pass

struct Geom {
  float sx2, sy2;         // (2/W)^2, (2/H)^2: squared NDC size of a pixel along columns / rows
  float r2;               // r^2 (NDC)
  float rx, ry;           // r in pixels along columns (r W / 2) and rows (r H / 2)
  int H, W, tiles_x, tiles_y;
};

__device__ __forceinline__ float ndc_d2(float col, float row, int j, int i, const Geom& g) {
  const float dx = __fsub_rn(col, (float)j), dy = __fsub_rn(row, (float)i);
  return __fadd_rn(__fmul_rn(g.sx2, __fmul_rn(dx, dx)), __fmul_rn(g.sy2, __fmul_rn(dy, dy)));
}

__device__ __forceinline__ float weight(float d2, float r2) { return __fsub_rn(1.f, __fdiv_rn(d2, r2)); }

// (Z, index) order as one unsigned key: Z >= 0, so its bit pattern orders like its value (-0 folded onto +0)
__device__ __forceinline__ unsigned long long point_key(float z, long long p) {
  return ((unsigned long long)__float_as_uint(z == 0.f ? 0.f : z) << 32) | (unsigned long long)p;
}

// Pixels [lo, hi] along one axis that a disc of half-width `rad` pixels centred at c may cover: |c - j| < rad,
// widened by one pixel on each side so that no pixel the fp32 test accepts is left out.  False when none is inside.
__device__ __forceinline__ bool pixel_range(float c, float rad, int n_px, int& lo, int& hi) {
  if (!(c + rad >= -1.f) || !(c - rad <= (float)n_px)) return false;      // also false for NaN
  lo = max(0, (int)floorf(fmaxf(c - rad, -2.f)));
  hi = min(n_px - 1, (int)ceilf(fminf(c + rad, (float)n_px + 1.f)));
  return lo <= hi;
}

__global__ void __launch_bounds__(256)
bin_kernel(const float* __restrict__ pts, const long long* __restrict__ order, long long N, long long V, Geom g,
           int tmax_x, int tmax_y, long long* __restrict__ keys, int* __restrict__ ids) {
  const int tmax = tmax_x * tmax_y;
  const long long sentinel = N * g.tiles_x * g.tiles_y;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < N * V;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long n = idx / V;
    const int p = (int)order[idx];
    const float* q = pts + (n * V + p) * 3;
    long long* k = keys + idx * tmax;
    int* d = ids + idx * tmax;
    int t = 0, c0, c1, r0, r1;
    if (q[2] >= 0.f && pixel_range(q[0], g.rx, g.W, c0, c1) && pixel_range(q[1], g.ry, g.H, r0, r1)) {
      const int tx0 = c0 / kTile, tx1 = min(c1 / kTile, tx0 + tmax_x - 1);
      const int ty0 = r0 / kTile, ty1 = min(r1 / kTile, ty0 + tmax_y - 1);
      for (int ty = ty0; ty <= ty1; ++ty)
        for (int tx = tx0; tx <= tx1; ++tx) {
          k[t] = (n * g.tiles_y + ty) * g.tiles_x + tx;
          d[t] = p;
          ++t;
        }
    }
    for (; t < tmax; ++t) {
      k[t] = sentinel;
      d[t] = -1;
    }
  }
}

__global__ void __launch_bounds__(kTile * kTile)
forward_kernel(const float* __restrict__ pts, const long long* __restrict__ offsets, const int* __restrict__ ids,
               long long V, Geom g, int K, float* __restrict__ mask, unsigned long long* __restrict__ kth,
               float* __restrict__ prod, int* __restrict__ zeros) {
  __shared__ float s_col[kChunk], s_row[kChunk];
  __shared__ unsigned long long s_key[kChunk];
  const int tile = blockIdx.x;
  const long long n = blockIdx.y;
  const int j = (tile % g.tiles_x) * kTile + (threadIdx.x % kTile);
  const int i = (tile / g.tiles_x) * kTile + (threadIdx.x / kTile);
  const bool inside = i < g.H && j < g.W;
  const long long t = n * g.tiles_x * g.tiles_y + tile;
  const long long b = offsets[t], e = offsets[t + 1];
  const float* P = pts + n * V * 3;
  int cnt = inside ? 0 : K;            // pixels outside the image count as full for the early exit
  float acc = 0.f, trans = 1.f, pnz = 1.f;
  int nz = 0;
  unsigned long long last = ~0ULL;
  for (long long c = b; c < e; c += kChunk) {
    if (__syncthreads_and(cnt >= K)) break;      // also the barrier before the chunk buffers are overwritten
    const long long m = c + threadIdx.x;
    if (m < e) {
      const long long p = ids[m];
      s_col[threadIdx.x] = P[p * 3];
      s_row[threadIdx.x] = P[p * 3 + 1];
      s_key[threadIdx.x] = point_key(P[p * 3 + 2], p);
    }
    __syncthreads();
    const int len = (int)min((long long)kChunk, e - c);
    for (int u = 0; u < len && cnt < K; ++u) {
      const float d2 = ndc_d2(s_col[u], s_row[u], j, i, g);
      if (d2 < g.r2) {
        const float w = weight(d2, g.r2);
        const float om = __fsub_rn(1.f, w);
        acc = __fadd_rn(acc, __fmul_rn(w, trans));
        trans = __fmul_rn(trans, om);
        if (om == 0.f) ++nz;
        else pnz = __fmul_rn(pnz, om);
        last = s_key[u];
        ++cnt;
      }
    }
  }
  if (inside) {
    const long long idx = (n * g.H + i) * g.W + j;
    mask[idx] = acc;
    kth[idx] = cnt >= K ? last : ~0ULL;
    prod[idx] = pnz;
    zeros[idx] = nz;
  }
}

__global__ void __launch_bounds__(256)
backward_kernel(const float* __restrict__ pts, const float* __restrict__ gmask,
                const unsigned long long* __restrict__ kth, const float* __restrict__ prod,
                const int* __restrict__ zeros, long long N, long long V, Geom g, float* __restrict__ gpts) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < N * V;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long n = idx / V, p = idx % V;
    const float col = pts[idx * 3], row = pts[idx * 3 + 1], z = pts[idx * 3 + 2];
    float gc = 0.f, gr = 0.f;
    int c0, c1, r0, r1;
    if (z >= 0.f && pixel_range(col, g.rx, g.W, c0, c1) && pixel_range(row, g.ry, g.H, r0, r1)) {
      const unsigned long long key = point_key(z, p);
      for (int i = r0; i <= r1; ++i)
        for (int j = c0; j <= c1; ++j) {
          const float d2 = ndc_d2(col, row, j, i, g);
          if (!(d2 < g.r2)) continue;
          const long long pix = (n * g.H + i) * g.W + j;
          if (key > kth[pix]) continue;                // covers the pixel but is not among its K kept points
          const float om = __fsub_rn(1.f, weight(d2, g.r2));
          const int nzp = zeros[pix];
          // prod_{q kept, q != p} (1 - w_q) from the pixel's product of nonzero factors and its zero count
          const float others = om == 0.f ? (nzp == 1 ? prod[pix] : 0.f) : (nzp == 0 ? prod[pix] / om : 0.f);
          const float gd2 = -(gmask[pix] * others) / g.r2;      // dL/dd2 = dL/dmask * dmask/dw * dw/dd2
          gc += gd2 * (2.f * g.sx2 * (col - (float)j));
          gr += gd2 * (2.f * g.sy2 * (row - (float)i));
        }
    }
    gpts[idx * 3] = gc;
    gpts[idx * 3 + 1] = gr;
    gpts[idx * 3 + 2] = 0.f;
  }
}

// Geometry and the per-point tile bound; false on invalid arguments.
bool make_geom(int64_t N, int64_t V, int H, int W, float radius, Geom& g, int& tmax_x, int& tmax_y) {
  if (N <= 0 || V <= 0 || V > 0x7fffffffLL || H <= 0 || W <= 0 || !(radius > 0.f) || !isfinite(radius)) return false;
  g.tiles_x = (W + kTile - 1) / kTile;
  g.tiles_y = (H + kTile - 1) / kTile;
  if ((double)N * g.tiles_x * g.tiles_y > 4e18) return false;
  const double rx = (double)radius * W / 2.0, ry = (double)radius * H / 2.0;
  g.rx = (float)rx;
  g.ry = (float)ry;
  g.sx2 = (float)((2.0 / W) * (2.0 / W));
  g.sy2 = (float)((2.0 / H) * (2.0 / H));
  g.r2 = (float)((double)radius * radius);
  g.H = H;
  g.W = W;
  // a point's pixel range spans at most 2 rad + 2 pixels (pixel_range), + 0.5 against fp32 rounding of c +- rad
  tmax_x = (int)fmin((double)g.tiles_x, floor((2.0 * rx + 2.5) / kTile) + 2.0);
  tmax_y = (int)fmin((double)g.tiles_y, floor((2.0 * ry + 2.5) / kTile) + 2.0);
  return (double)N * V * tmax_x * tmax_y < 4e18;
}

}  // namespace

extern "C" int64_t sr_points_silhouette_list_capacity(int64_t N, int64_t V, int H, int W, float radius) {
  Geom g;
  int tx, ty;
  if (!make_geom(N, V, H, W, radius, g, tx, ty)) return SR_EINVAL;
  return N * V * tx * ty;
}

extern "C" int sr_points_silhouette_bin(const float* pts_screen, const int64_t* order, int64_t N, int64_t V, int H,
                                        int W, float radius, int64_t* tile_keys, int32_t* tile_points,
                                        cudaStream_t s) {
  Geom g;
  int tx, ty;
  if (!pts_screen || !order || !tile_keys || !tile_points || !make_geom(N, V, H, W, radius, g, tx, ty))
    return SR_EINVAL;
  bin_kernel<<<sr_grid_for(N * V, 256, 8), 256, 0, s>>>(pts_screen, (const long long*)order, N, V, g, tx, ty,
                                                        (long long*)tile_keys, (int*)tile_points);
  return sr_launch_status();
}

extern "C" int sr_points_silhouette_forward(const float* pts_screen, const int64_t* tile_offsets,
                                            const int32_t* tile_points, int64_t N, int64_t V, int H, int W,
                                            float radius, int K, float* mask, uint64_t* kth_key, float* prod,
                                            int32_t* zeros, cudaStream_t s) {
  Geom g;
  int tx, ty;
  if (!pts_screen || !tile_offsets || !tile_points || !mask || !kth_key || !prod || !zeros || K <= 0 ||
      !make_geom(N, V, H, W, radius, g, tx, ty) || N > 65535)
    return SR_EINVAL;
  const dim3 grid((unsigned)(g.tiles_x * g.tiles_y), (unsigned)N);
  forward_kernel<<<grid, kTile * kTile, 0, s>>>(pts_screen, (const long long*)tile_offsets, (const int*)tile_points,
                                                V, g, K, mask, (unsigned long long*)kth_key, prod, (int*)zeros);
  return sr_launch_status();
}

extern "C" int sr_points_silhouette_backward(const float* pts_screen, const float* grad_mask, const uint64_t* kth_key,
                                             const float* prod, const int32_t* zeros, int64_t N, int64_t V, int H,
                                             int W, float radius, float* grad_pts, cudaStream_t s) {
  Geom g;
  int tx, ty;
  if (!pts_screen || !grad_mask || !kth_key || !prod || !zeros || !grad_pts || !make_geom(N, V, H, W, radius, g, tx, ty))
    return SR_EINVAL;
  backward_kernel<<<sr_grid_for(N * V, 256, 8), 256, 0, s>>>(pts_screen, grad_mask,
                                                             (const unsigned long long*)kth_key, prod, (const int*)zeros,
                                                             N, V, g, grad_pts);
  return sr_launch_status();
}
