// Chart segmentation, projection and overlap check of the UV atlas of a template mesh (uvmap.unwrap).
//   directions  the 26 d_L = normalize(i, j, k), (i, j, k) in {-1, 0, 1}^3 \ 0 in lexicographic order (i slowest).
//   adjacency   adj[3f+k] = the other face across the edge opposite corner k when that edge has exactly two faces,
//               else -1 (a scan of the first corner's vertex -> face CSR).
//   labels      argmax_L n_f . d_L, lowest L on ties; a zero-area face takes the label of its lowest-id neighbour
//               with a normal (0 without one).  Smoothing pass (Jacobi): among the labels L of f and its neighbours
//               with n_f . d_L >= cos(max_angle), the one whose faces in {f, neighbours} have the largest summed area
//               (summed in the order f, adj[3f], adj[3f+1], adj[3f+2]), lowest L on ties; no candidate keeps f's label.
//   charts      connected components of same-label faces across two-face edges; id = minimum face id, found by
//               repeated in-place hooking to the smallest id seen plus one pointer jump, until no id changes (the
//               fixed point does not depend on the schedule).
//   projection  one block per chart, over its (chart, vertex) UV vertices: (p . t1, p . t2) with t1 = normalize(d x
//               e_k), k = d's smallest-|component| axis (lowest k on ties), t2 = d x t1; rotated by -theta, theta =
//               atan2(2 c_xy, c_xx - c_yy) / 2 of the vertices' covariance, then by +90 degrees when taller than wide,
//               and shifted to a zero minimum.  fp64, fixed-order block sums.
//   coverage    per UV face the texel centres (col, row) of the bake's raster (x = u R - 0.5, y = (1 - v) R - 0.5)
//               inside it under a half-open rule: edge functions in fp64 from the fp32 UVs, each evaluated from the
//               edge's lexicographically smaller end (no FMA), and a centre on an edge belongs to the face when the
//               edge, taken in the face's positive orientation, points down (+y) or, horizontal, right.  Integer
//               atomic counts: bit-identical reruns.
// All passes are gathers over short lists or per-face bounding-box walks: latency / L2 bound.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kDirs = 26;

__device__ __forceinline__ double3 ld3(const float* __restrict__ v, long long i) {
  return make_double3((double)v[3 * i], (double)v[3 * i + 1], (double)v[3 * i + 2]);
}
__device__ __forceinline__ double3 sub(double3 a, double3 b) { return make_double3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double dot(double3 a, double3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ double3 cross(double3 a, double3 b) {
  return make_double3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

__device__ __forceinline__ double3 direction(int L) {
  const int t = L < 13 ? L : L + 1;
  const double i = t / 9 - 1, j = (t / 3) % 3 - 1, k = t % 3 - 1;
  const double r = sqrt(i * i + j * j + k * k);
  return make_double3(i / r, j / r, k / r);
}

__device__ __forceinline__ int argmax_label(double3 n) {
  int best = 0;
  double bd = dot(n, direction(0));
  for (int L = 1; L < kDirs; ++L) {
    const double d = dot(n, direction(L));
    if (d > bd) { bd = d; best = L; }
  }
  return best;
}

__device__ __forceinline__ double3 face_normal(const float* __restrict__ verts, const long long* __restrict__ f) {
  const double3 p0 = ld3(verts, f[0]);
  return cross(sub(ld3(verts, f[1]), p0), sub(ld3(verts, f[2]), p0));
}

__global__ void __launch_bounds__(kThreads)
adjacency_kernel(const long long* __restrict__ faces, long long F, const long long* __restrict__ vf_off,
                 const long long* __restrict__ vf, long long* __restrict__ adj) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < 3 * F;
       t += (long long)gridDim.x * blockDim.x) {
    const long long f = t / 3, k = t % 3;
    const long long a = faces[3 * f + (k + 1) % 3], b = faces[3 * f + (k + 2) % 3];
    long long other = -1, m = 0;
    for (long long i = vf_off[a]; i < vf_off[a + 1]; ++i) {
      const long long g = vf[i];
      if (g == f) continue;
      const long long* q = faces + 3 * g;
      if (q[0] == b || q[1] == b || q[2] == b) { other = g; ++m; }
    }
    adj[t] = m == 1 ? other : -1;
  }
}

__global__ void __launch_bounds__(kThreads)
label_init_kernel(const float* __restrict__ verts, const long long* __restrict__ faces, long long F,
                  const long long* __restrict__ adj, double* __restrict__ normal, double* __restrict__ area,
                  int32_t* __restrict__ label) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    const double3 n = face_normal(verts, faces + 3 * f);
    const double len = sqrt(dot(n, n));
    double3 u = make_double3(0.0, 0.0, 0.0);
    int L = 0;
    if (len > 0.0) {
      u = make_double3(n.x / len, n.y / len, n.z / len);
      L = argmax_label(u);
    } else {
      long long best = -1;
      for (int k = 0; k < 3; ++k) {
        const long long g = adj[3 * f + k];
        if (g < 0 || (best >= 0 && g >= best)) continue;
        const double3 m = face_normal(verts, faces + 3 * g);
        if (dot(m, m) > 0.0) best = g;
      }
      if (best >= 0) {
        const double3 m = face_normal(verts, faces + 3 * best);
        const double ml = sqrt(dot(m, m));
        L = argmax_label(make_double3(m.x / ml, m.y / ml, m.z / ml));
      }
    }
    normal[3 * f] = u.x;
    normal[3 * f + 1] = u.y;
    normal[3 * f + 2] = u.z;
    area[f] = 0.5 * len;
    label[f] = L;
  }
}

__global__ void __launch_bounds__(kThreads)
label_smooth_kernel(const double* __restrict__ normal, const double* __restrict__ area,
                    const long long* __restrict__ adj, long long F, double cos_max, const int32_t* __restrict__ in,
                    int32_t* __restrict__ out) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    long long ids[4] = {f, adj[3 * f], adj[3 * f + 1], adj[3 * f + 2]};
    int lab[4];
    for (int i = 0; i < 4; ++i) lab[i] = ids[i] >= 0 ? in[ids[i]] : -1;
    const double3 n = make_double3(normal[3 * f], normal[3 * f + 1], normal[3 * f + 2]);
    int best = in[f];
    double bs = -1.0;
    for (int c = 0; c < 4; ++c) {
      const int L = lab[c];
      if (L < 0 || dot(n, direction(L)) < cos_max) continue;
      double s = 0.0;
      for (int i = 0; i < 4; ++i)
        if (lab[i] == L) s += area[ids[i]];
      if (s > bs || (s == bs && L < best)) { bs = s; best = L; }
    }
    out[f] = best;
  }
}

__global__ void __launch_bounds__(kThreads)
chart_hook_kernel(const long long* __restrict__ adj, const int32_t* __restrict__ label, long long F,
                  long long* __restrict__ cid, int32_t* __restrict__ changed) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    volatile long long* c = cid;
    long long m = c[f];
    for (int k = 0; k < 3; ++k) {
      const long long g = adj[3 * f + k];
      if (g >= 0 && label[g] == label[f]) m = min(m, c[g]);
    }
    m = min(m, c[m]);
    if (m < c[f]) {
      c[f] = m;
      *changed = 1;
    }
  }
}

// Fixed-order block reductions (thread 0's partials first, then warp by warp).
template <int N, typename Op>
__device__ __forceinline__ void block_reduce(double v[N], Op op) {
  __shared__ double red[N][kThreads / 32];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < N; ++c) {
    for (int o = 16; o > 0; o >>= 1) v[c] = op(v[c], __shfl_xor_sync(0xffffffffu, v[c], o));
    if (l == 0) red[c][w] = v[c];
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < N; ++c) {
    double s = red[c][0];
    for (int k = 1; k < kThreads / 32; ++k) s = op(s, red[c][k]);
    v[c] = s;
  }
  __syncthreads();
}

struct Add { __device__ double operator()(double a, double b) const { return a + b; } };
struct Min { __device__ double operator()(double a, double b) const { return fmin(a, b); } };

__global__ void __launch_bounds__(kThreads)
chart_project_kernel(const float* __restrict__ verts, long long C, const long long* __restrict__ chart_off,
                     const long long* __restrict__ uv_vert, const int32_t* __restrict__ chart_label,
                     double* __restrict__ uvl, double* __restrict__ box) {
  for (long long ch = blockIdx.x; ch < C; ch += gridDim.x) {
    const long long i0 = chart_off[ch], i1 = chart_off[ch + 1];
    const double3 d = direction(chart_label[ch]);
    const double ad[3] = {fabs(d.x), fabs(d.y), fabs(d.z)};
    const int k = ad[0] <= ad[1] && ad[0] <= ad[2] ? 0 : (ad[1] <= ad[2] ? 1 : 2);
    const double3 ek = make_double3(k == 0, k == 1, k == 2);
    double3 t1 = cross(d, ek);
    const double r = sqrt(dot(t1, t1));
    t1 = make_double3(t1.x / r, t1.y / r, t1.z / r);
    const double3 t2 = cross(d, t1);
    double s[2] = {0.0, 0.0};
    for (long long i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
      const double3 p = ld3(verts, uv_vert[i]);
      const double x = dot(p, t1), y = dot(p, t2);
      uvl[2 * i] = x;
      uvl[2 * i + 1] = y;
      s[0] += x;
      s[1] += y;
    }
    block_reduce<2>(s, Add());
    const double n = (double)(i1 - i0), mx = s[0] / n, my = s[1] / n;
    double cv[3] = {0.0, 0.0, 0.0};
    for (long long i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
      const double x = uvl[2 * i] - mx, y = uvl[2 * i + 1] - my;
      cv[0] += x * x;
      cv[1] += x * y;
      cv[2] += y * y;
    }
    block_reduce<3>(cv, Add());
    const double th = 0.5 * atan2(2.0 * cv[1], cv[0] - cv[2]), c = cos(th), sn = sin(th);
    // rotated (u, v) = R(-theta) (x - mx, y - my); bounds as minima of (u, -u, v, -v)
    double b[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
    for (long long i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
      const double x = uvl[2 * i] - mx, y = uvl[2 * i + 1] - my;
      const double u = c * x + sn * y, v = -sn * x + c * y;
      b[0] = fmin(b[0], u); b[1] = fmin(b[1], -u); b[2] = fmin(b[2], v); b[3] = fmin(b[3], -v);
    }
    block_reduce<4>(b, Min());
    const double w = -b[1] - b[0], h = -b[3] - b[2];
    const bool turn = h > w;   // +90 degrees: (u, v) -> (-v, u)
    for (long long i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
      const double x = uvl[2 * i] - mx, y = uvl[2 * i + 1] - my;
      const double u = c * x + sn * y, v = -sn * x + c * y;
      uvl[2 * i] = turn ? -v - b[3] : u - b[0];
      uvl[2 * i + 1] = turn ? u - b[0] : v - b[2];
    }
    if (threadIdx.x == 0) {
      box[2 * ch] = turn ? h : w;
      box[2 * ch + 1] = turn ? w : h;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kThreads)
place_kernel(const double* __restrict__ uvl, const long long* __restrict__ uv_chart, long long T,
             const double* __restrict__ offset, double scale, float* __restrict__ vt) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < T; i += (long long)gridDim.x * blockDim.x) {
    const long long c = uv_chart[i];
    vt[2 * i] = (float)(offset[2 * c] + scale * uvl[2 * i]);
    vt[2 * i + 1] = (float)(offset[2 * c + 1] + scale * uvl[2 * i + 1]);
  }
}

// (q - p) x (t - p) with no contraction, evaluated from the lexicographically smaller end so that the two faces of a
// shared edge compute the same magnitude.
__device__ __forceinline__ double edge_fn(double px, double py, double qx, double qy, double tx, double ty) {
  const bool swap = qx < px || (qx == px && qy < py);
  const double ax = swap ? qx : px, ay = swap ? qy : py, bx = swap ? px : qx, by = swap ? py : qy;
  const double w = __dsub_rn(__dmul_rn(__dsub_rn(bx, ax), __dsub_rn(ty, ay)),
                             __dmul_rn(__dsub_rn(by, ay), __dsub_rn(tx, ax)));
  return swap ? -w : w;
}

struct UvTri {
  double x[3], y[3], sgn;
  int c0, c1, r0, r1;
};

__device__ __forceinline__ bool load_uv_tri(const float* __restrict__ vt, const long long* __restrict__ ft,
                                            long long f, int R, UvTri& t) {
  for (int k = 0; k < 3; ++k) {
    const long long i = ft[3 * f + k];
    t.x[k] = __dsub_rn(__dmul_rn((double)vt[2 * i], (double)R), 0.5);
    t.y[k] = __dsub_rn(__dmul_rn(__dsub_rn(1.0, (double)vt[2 * i + 1]), (double)R), 0.5);
  }
  const double a = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], t.x[2], t.y[2]);
  if (a == 0.0) return false;
  t.sgn = a > 0.0 ? 1.0 : -1.0;
  t.c0 = max(0, (int)ceil(fmin(t.x[0], fmin(t.x[1], t.x[2]))));
  t.c1 = min(R - 1, (int)floor(fmax(t.x[0], fmax(t.x[1], t.x[2]))));
  t.r0 = max(0, (int)ceil(fmin(t.y[0], fmin(t.y[1], t.y[2]))));
  t.r1 = min(R - 1, (int)floor(fmax(t.y[0], fmax(t.y[1], t.y[2]))));
  return true;
}

__device__ __forceinline__ bool covers(const UvTri& t, double cx, double cy) {
  for (int k = 0; k < 3; ++k) {
    const int j = (k + 1) % 3;
    const double w = t.sgn * edge_fn(t.x[k], t.y[k], t.x[j], t.y[j], cx, cy);
    if (w < 0.0) return false;
    if (w == 0.0) {
      const double dx = t.sgn * (t.x[j] - t.x[k]), dy = t.sgn * (t.y[j] - t.y[k]);
      if (!(dy > 0.0 || (dy == 0.0 && dx > 0.0))) return false;
    }
  }
  return true;
}

__global__ void __launch_bounds__(kThreads)
coverage_kernel(const float* __restrict__ vt, const long long* __restrict__ ft, long long F, int R,
                int32_t* __restrict__ count) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    UvTri t;
    if (!load_uv_tri(vt, ft, f, R, t)) continue;
    for (int r = t.r0; r <= t.r1; ++r)
      for (int c = t.c0; c <= t.c1; ++c)
        if (covers(t, (double)c, (double)r)) atomicAdd(&count[(long long)r * R + c], 1);
  }
}

__global__ void __launch_bounds__(kThreads)
overlap_faces_kernel(const float* __restrict__ vt, const long long* __restrict__ ft, long long F, int R,
                     const int32_t* __restrict__ count, uint8_t* __restrict__ bad) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    UvTri t;
    bool b = false;
    if (load_uv_tri(vt, ft, f, R, t))
      for (int r = t.r0; r <= t.r1 && !b; ++r)
        for (int c = t.c0; c <= t.c1 && !b; ++c)
          b = count[(long long)r * R + c] > 1 && covers(t, (double)c, (double)r);
    bad[f] = b;
  }
}

}  // namespace

extern "C" int sr_uv_face_adjacency(const int64_t* faces, int64_t F, const int64_t* vf_off, const int64_t* vf,
                                    int64_t* adj, cudaStream_t s) {
  if (!faces || !vf_off || !vf || !adj || F <= 0) return SR_EINVAL;
  adjacency_kernel<<<sr_grid_for(3 * F, kThreads, 8), kThreads, 0, s>>>(
      (const long long*)faces, F, (const long long*)vf_off, (const long long*)vf, (long long*)adj);
  return sr_launch_status();
}

extern "C" int sr_uv_labels(const float* verts, const int64_t* faces, int64_t F, const int64_t* adj, float max_angle,
                            int passes, double* normal, double* area, int32_t* label, int32_t* work, cudaStream_t s) {
  if (!verts || !faces || !adj || !normal || !area || !label || !work || F <= 0 || passes < 0 ||
      !(max_angle >= 35.f && max_angle <= 80.f))
    return SR_EINVAL;
  const int grid = sr_grid_for(F, kThreads, 8);
  const double cos_max = cos((double)max_angle * 3.14159265358979323846 / 180.0);
  label_init_kernel<<<grid, kThreads, 0, s>>>(verts, (const long long*)faces, F, (const long long*)adj, normal, area,
                                              passes % 2 ? work : label);
  for (int p = 0; p < passes; ++p) {
    const bool into_label = (passes - p) % 2 == 1;   // the last pass writes `label`
    label_smooth_kernel<<<grid, kThreads, 0, s>>>(normal, area, (const long long*)adj, F, cos_max,
                                                  into_label ? work : label, into_label ? label : work);
  }
  return sr_launch_status();
}

extern "C" int sr_uv_chart_hook(const int64_t* adj, const int32_t* label, int64_t F, int64_t* cid, int32_t* changed,
                                cudaStream_t s) {
  if (!adj || !label || !cid || !changed || F <= 0) return SR_EINVAL;
  cudaError_t e = cudaMemsetAsync(changed, 0, 4, s);
  if (e != cudaSuccess) return (int)e;
  chart_hook_kernel<<<sr_grid_for(F, kThreads, 8), kThreads, 0, s>>>((const long long*)adj, label, F,
                                                                      (long long*)cid, changed);
  return sr_launch_status();
}

extern "C" int sr_uv_chart_project(const float* verts, int64_t C, const int64_t* chart_off, const int64_t* uv_vert,
                                   const int32_t* chart_label, double* uvl, double* box, cudaStream_t s) {
  if (!verts || !chart_off || !uv_vert || !chart_label || !uvl || !box || C <= 0) return SR_EINVAL;
  const int grid = (int)(C < 8 * SR_NUM_SMS ? C : 8 * SR_NUM_SMS);
  chart_project_kernel<<<grid, kThreads, 0, s>>>(verts, C, (const long long*)chart_off, (const long long*)uv_vert,
                                                 chart_label, uvl, box);
  return sr_launch_status();
}

extern "C" int sr_uv_place(const double* uvl, const int64_t* uv_chart, int64_t T, const double* offset, double scale,
                           float* vt, cudaStream_t s) {
  if (!uvl || !uv_chart || !offset || !vt || T <= 0 || !(scale > 0.0)) return SR_EINVAL;
  place_kernel<<<sr_grid_for(T, kThreads, 8), kThreads, 0, s>>>(uvl, (const long long*)uv_chart, T, offset, scale,
                                                                vt);
  return sr_launch_status();
}

extern "C" int sr_uv_coverage(const float* vt, const int64_t* ft, int64_t F, int R, int32_t* count, uint8_t* bad,
                              cudaStream_t s) {
  if (!vt || !ft || !count || F <= 0 || R <= 0) return SR_EINVAL;
  cudaError_t e = cudaMemsetAsync(count, 0, (size_t)R * R * 4, s);
  if (e != cudaSuccess) return (int)e;
  const int grid = sr_grid_for(F, kThreads, 8);
  coverage_kernel<<<grid, kThreads, 0, s>>>(vt, (const long long*)ft, F, R, count);
  if (bad) overlap_faces_kernel<<<grid, kThreads, 0, s>>>(vt, (const long long*)ft, F, R, count, bad);
  return sr_launch_status();
}
