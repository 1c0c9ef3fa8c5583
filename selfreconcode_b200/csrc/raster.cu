// Device-side mesh rasteriser for the ray seed (SURVEY.md section 8f-1): replaces the pytorch3d MeshRasterizer call
// whose fragments feed utils.FindSurfacePs (model/network.py:492, 345; utils/FindSurfacePs.py:5-29).
// Input: per frame, vertices already projected by the camera to pixel coordinates (x = column, y = row, pixel centres
// at integers -- RectifiedPerspectiveCameras.project, model/CameraMine.py:138-142) plus the camera-space depth z.
// Output (pytorch3d's Fragments with faces_per_pixel = 1, blur_radius = 0, perspective_correct = True,
// clip_barycentric_coords = False, cull_backfaces = False):
//   pix_to_face [N,H,W] int64: n*F + f of the nearest covering face, -1 where none
//   bary        [N,H,W,3] perspective-correct barycentrics of the pixel centre in that face (-1 where none)
//   zbuf        [N,H,W] interpolated depth (-1 where none)
// Two kernels: (1) one thread per (frame, face) walks the face's pixel bounding box and atomicMin's a 64-bit
// (depth bits, face id) key per covered pixel; (2) one thread per pixel decodes the winner and recomputes its
// barycentrics.  HBM-bound on the 8-byte key image (8 B/pixel written + read) and 36 B per face read.
#include "common.cuh"

namespace {

struct Tri {
  float x0, y0, z0, x1, y1, z1, x2, y2, z2;
};

__device__ __forceinline__ bool load_tri(const float* __restrict__ vs, const long long* __restrict__ faces,
                                         long long n, long long V, long long f, Tri& t) {
  const long long a = faces[f * 3], b = faces[f * 3 + 1], c = faces[f * 3 + 2];
  const float* p = vs + n * V * 3;
  t.x0 = p[a * 3]; t.y0 = p[a * 3 + 1]; t.z0 = p[a * 3 + 2];
  t.x1 = p[b * 3]; t.y1 = p[b * 3 + 1]; t.z1 = p[b * 3 + 2];
  t.x2 = p[c * 3]; t.y2 = p[c * 3 + 1]; t.z2 = p[c * 3 + 2];
  // a non-finite vertex drops the face: with z = inf its q_i would be 0 and the face would still cover pixels
  const bool finite = isfinite(t.x0) && isfinite(t.y0) && isfinite(t.z0) && isfinite(t.x1) && isfinite(t.y1) &&
                      isfinite(t.z1) && isfinite(t.x2) && isfinite(t.y2) && isfinite(t.z2);
  return finite && t.z0 > 1e-8f && t.z1 > 1e-8f && t.z2 > 1e-8f;
}

// Edge function of the directed edge a -> b at (px, py): (xa - px)(yb - py) - (xb - px)(ya - py), twice the signed
// area of (a, b, p).  Every difference and product is rounded on its own: __fmul_rn / __fsub_rn are never contracted
// into an FFMA, so edge(a, b) == -edge(b, a) bit for bit.  Two faces sharing an edge then cannot both reject a pixel
// centre on it (the coverage test is watertight), a face's coverage does not depend on its winding, and the face and
// resolve kernels take the same decision on the same pixel.  It is also the face area: area = edge(v1, v2) at v0.
__device__ __forceinline__ float edge_fn(float xa, float ya, float xb, float yb, float px, float py) {
  return __fsub_rn(__fmul_rn(__fsub_rn(xa, px), __fsub_rn(yb, py)), __fmul_rn(__fsub_rn(xb, px), __fsub_rn(ya, py)));
}

// barycentrics of pixel centre (px, py); returns false when outside or degenerate
__device__ __forceinline__ bool bary_at(const Tri& t, float px, float py, float b[3], float& z) {
  const float area = edge_fn(t.x1, t.y1, t.x2, t.y2, t.x0, t.y0);
  if (fabsf(area) < 1e-12f) return false;
  const float w0 = edge_fn(t.x1, t.y1, t.x2, t.y2, px, py);
  const float w1 = edge_fn(t.x2, t.y2, t.x0, t.y0, px, py);
  const float w2 = edge_fn(t.x0, t.y0, t.x1, t.y1, px, py);
  const float inv = 1.0f / area;
  const float l0 = w0 * inv, l1 = w1 * inv, l2 = w2 * inv;
  if (l0 < 0.f || l1 < 0.f || l2 < 0.f) return false;
  // perspective correction
  const float q0 = l0 / t.z0, q1 = l1 / t.z1, q2 = l2 / t.z2;
  const float s = q0 + q1 + q2;
  if (!(s > 0.f)) return false;
  b[0] = q0 / s; b[1] = q1 / s; b[2] = q2 / s;
  z = 1.0f / s;
  return true;
}

__global__ void __launch_bounds__(256)
raster_faces_kernel(const float* __restrict__ vs, const long long* __restrict__ faces, long long N, long long V,
                    long long F, int H, int W, unsigned long long* __restrict__ keys) {
  const long long total = N * F;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long n = idx / F, f = idx % F;
    Tri t;
    if (!load_tri(vs, faces, n, V, f, t)) continue;
    const float xmin = fminf(t.x0, fminf(t.x1, t.x2)), xmax = fmaxf(t.x0, fmaxf(t.x1, t.x2));
    const float ymin = fminf(t.y0, fminf(t.y1, t.y2)), ymax = fmaxf(t.y0, fmaxf(t.y1, t.y2));
    const int c0 = max(0, (int)ceilf(xmin)), c1 = min(W - 1, (int)floorf(xmax));
    const int r0 = max(0, (int)ceilf(ymin)), r1 = min(H - 1, (int)floorf(ymax));
    for (int r = r0; r <= r1; ++r)
      for (int c = c0; c <= c1; ++c) {
        float b[3], z;
        if (!bary_at(t, (float)c, (float)r, b, z)) continue;
        const unsigned long long key = ((unsigned long long)__float_as_uint(z) << 32) | (unsigned long long)f;
        atomicMin(&keys[(n * H + r) * W + c], key);
      }
  }
}

__global__ void __launch_bounds__(256)
raster_resolve_kernel(const float* __restrict__ vs, const long long* __restrict__ faces, long long N, long long V,
                      long long F, int H, int W, const unsigned long long* __restrict__ keys,
                      long long* __restrict__ pix_to_face, float* __restrict__ bary, float* __restrict__ zbuf) {
  const long long total = N * H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = keys[idx];
    long long out = -1;
    float b[3] = {-1.f, -1.f, -1.f}, z = -1.f;
    if (key != ~0ULL) {
      const long long n = idx / ((long long)H * W);
      const int r = (int)((idx / W) % H), c = (int)(idx % W);
      const long long f = (long long)(key & 0xffffffffULL);
      Tri t;
      load_tri(vs, faces, n, V, f, t);
      bary_at(t, (float)c, (float)r, b, z);
      out = n * F + f;
    }
    pix_to_face[idx] = out;
    bary[idx * 3] = b[0]; bary[idx * 3 + 1] = b[1]; bary[idx * 3 + 2] = b[2];
    if (zbuf) zbuf[idx] = z;
  }
}

}  // namespace

extern "C" int sr_raster_mesh(const float* verts_screen, const int64_t* faces, int64_t N, int64_t V, int64_t F,
                              int H, int W, uint64_t* keys, int64_t* pix_to_face, float* bary, float* zbuf,
                              cudaStream_t s) {
  if (!verts_screen || !faces || !keys || !pix_to_face || !bary || N <= 0 || V <= 0 || F <= 0 || H <= 0 || W <= 0 ||
      F > 0xffffffffLL)
    return SR_EINVAL;
  cudaError_t e = cudaMemsetAsync(keys, 0xff, (size_t)N * H * W * 8, s);
  if (e != cudaSuccess) return (int)e;
  raster_faces_kernel<<<sr_grid_for(N * F, 256, 8), 256, 0, s>>>(verts_screen, (const long long*)faces, N, V, F, H, W,
                                                                (unsigned long long*)keys);
  int rc = sr_launch_status();
  if (rc) return rc;
  raster_resolve_kernel<<<sr_grid_for(N * (long long)H * W, 256, 8), 256, 0, s>>>(
      verts_screen, (const long long*)faces, N, V, F, H, W, (const unsigned long long*)keys, (long long*)pix_to_face,
      bary, zbuf);
  return sr_launch_status();
}
