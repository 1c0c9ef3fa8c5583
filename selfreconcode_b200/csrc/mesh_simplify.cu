// Parallel quadric edge collapse of a reconstructed template (uvmap.simplify).  One round, over the edge table of
// csrc/mesh_reg.cu (edges [E,2] with a < b, the directed neighbour CSR, ascending) and the vertex -> face CSR
// (model.raster.vertex_face_csr, ascending face ids):
//   quadrics   Q_v = sum over v's CSR faces, in CSR order, of area * p p^T, p = (n, -n . v0) the face's unit plane;
//              fp64 from the fp32 positions.  A face of zero area adds nothing.
//   fixed      v is fixed when one of its edges has a face count other than 2, one of its faces repeats an index, or
//              its faces do not form one closed fan (the walk around the fan from its first face does not visit every
//              incident face; with two faces on every edge this also gives #faces = #edges).  Fixed vertices never
//              move and no edge touching one collapses.
//   cost       Q = Q_a + Q_b = [A b; b^T c].  When det A > 1e-6 (tr A / 3)^3 the position is v* = -A^-1 b (adjugate),
//              else the best of v_a, v_b and the midpoint in that order (strictly smaller cost wins).  The cost is
//              v*^T Q v* clamped at 0.
//   valid      neither end fixed; |N(a) n N(b)| = 2 (link condition); both opposite vertices have degree >= 4 (>= 3
//              after the collapse); every face around a or b that does not hold both keeps a non-zero normal that
//              turns by less than 90 degrees when its a or b corner moves to fp32(v*).
//   key        valid: (bits of fp32(cost) << 32) | e, else ~0.  m1(v) = min key over v's edges (integer atomicMin),
//              m2(v) = min of m1 over v and its neighbours; e is selected when key = m2(a) = m2(b) != ~0, so the
//              one-rings of two selected edges share no face and every check made on the old mesh still holds.
//   collapse   for a selected (a, b): b maps to a and a moves to fp32(v*); a face whose remapped corners repeat is
//              removed (exactly the two faces on the edge).  The caller's prefix sums of the alive flags compact
//              faces and vertices in ascending order.
// Every pass is a gather over short lists (~6 faces and ~6 neighbours per vertex): latency / L2 bound, as
// mesh_reg.cu.  The only atomics are the integer minima of the selection: bit-identical reruns.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr double kSingularRel = 1e-6;   // det A relative to (tr A / 3)^3 below which the 3x3 solve is not used
constexpr unsigned long long kNoKey = ~0ULL;

__device__ __forceinline__ double3 ld3(const float* __restrict__ v, long long i) {
  return make_double3((double)v[3 * i], (double)v[3 * i + 1], (double)v[3 * i + 2]);
}
__device__ __forceinline__ double3 sub(double3 a, double3 b) { return make_double3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double dot(double3 a, double3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ double3 cross(double3 a, double3 b) {
  return make_double3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

__device__ __forceinline__ bool has(const long long* __restrict__ f, long long v) {
  return f[0] == v || f[1] == v || f[2] == v;
}

__global__ void __launch_bounds__(kThreads)
quadrics_kernel(const float* __restrict__ verts, const long long* __restrict__ faces, long long V,
                const long long* __restrict__ vf_off, const long long* __restrict__ vf,
                const long long* __restrict__ nbr_off, const long long* __restrict__ nbr, double* __restrict__ Q,
                uint8_t* __restrict__ fixed) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    const long long f0 = vf_off[v], f1 = vf_off[v + 1];
    double q[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    bool fix = f1 == f0;
    for (long long i = f0; i < f1; ++i) {
      const long long* f = faces + 3 * vf[i];
      if (f[0] == f[1] || f[1] == f[2] || f[0] == f[2]) fix = true;
      const double3 p0 = ld3(verts, f[0]);
      const double3 n = cross(sub(ld3(verts, f[1]), p0), sub(ld3(verts, f[2]), p0));
      const double len = sqrt(dot(n, n));
      if (len == 0.0) continue;
      const double area = 0.5 * len, nx = n.x / len, ny = n.y / len, nz = n.z / len;
      const double d = -(nx * p0.x + ny * p0.y + nz * p0.z);
      const double p[4] = {nx, ny, nz, d};
      int k = 0;
      for (int r = 0; r < 4; ++r)
        for (int c = r; c < 4; ++c) q[k++] += area * p[r] * p[c];
    }
    for (int k = 0; k < 10; ++k) Q[10 * v + k] = q[k];
    // every edge at v has exactly two faces
    for (long long j = nbr_off[v]; j < nbr_off[v + 1] && !fix; ++j) {
      int m = 0;
      for (long long i = f0; i < f1; ++i) m += has(faces + 3 * vf[i], nbr[j]);
      fix = m != 2;
    }
    // one closed fan: walk from the first face across its edges at v
    if (!fix) {
      const long long* f = faces + 3 * vf[f0];
      const int kv = f[0] == v ? 0 : (f[1] == v ? 1 : 2);
      long long cur = vf[f0], x = f[(kv + 1) % 3];
      long long n = 0;
      do {
        long long nxt = -1;
        for (long long i = f0; i < f1; ++i)
          if (vf[i] != cur && has(faces + 3 * vf[i], x)) { nxt = vf[i]; break; }
        if (nxt < 0) break;
        const long long* g = faces + 3 * nxt;
        x = g[0] != v && g[0] != x ? g[0] : (g[1] != v && g[1] != x ? g[1] : g[2]);
        cur = nxt;
        ++n;
      } while (cur != vf[f0] && n <= f1 - f0);
      fix = n != f1 - f0;
    }
    fixed[v] = fix;
  }
}

__device__ __forceinline__ double qeval(const double* q, double3 v) {
  // [v 1] Q [v 1]^T with Q = [q0 q1 q2 q3; . q4 q5 q6; . . q7 q8; . . . q9]
  return q[0] * v.x * v.x + q[4] * v.y * v.y + q[7] * v.z * v.z + 2.0 * (q[1] * v.x * v.y + q[2] * v.x * v.z +
         q[5] * v.y * v.z) + 2.0 * (q[3] * v.x + q[6] * v.y + q[8] * v.z) + q[9];
}

__global__ void __launch_bounds__(kThreads)
edge_cost_kernel(const float* __restrict__ verts, const long long* __restrict__ faces,
                 const long long* __restrict__ edges, long long E, const long long* __restrict__ vf_off,
                 const long long* __restrict__ vf, const long long* __restrict__ nbr_off,
                 const long long* __restrict__ nbr, const double* __restrict__ Q, const uint8_t* __restrict__ fixed,
                 double* __restrict__ vstar, double* __restrict__ cost, unsigned long long* __restrict__ key) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    const long long a = edges[2 * e], b = edges[2 * e + 1];
    double q[10];
    for (int k = 0; k < 10; ++k) q[k] = Q[10 * a + k] + Q[10 * b + k];
    const double3 pa = ld3(verts, a), pb = ld3(verts, b);
    // adjugate of A = [q0 q1 q2; q1 q4 q5; q2 q5 q7]
    const double c00 = q[4] * q[7] - q[5] * q[5], c01 = q[2] * q[5] - q[1] * q[7], c02 = q[1] * q[5] - q[2] * q[4];
    const double c11 = q[0] * q[7] - q[2] * q[2], c12 = q[1] * q[2] - q[0] * q[5], c22 = q[0] * q[4] - q[1] * q[1];
    const double det = q[0] * c00 + q[1] * c01 + q[2] * c02;
    const double t3 = (q[0] + q[4] + q[7]) / 3.0;
    double3 v;
    double c;
    if (t3 > 0.0 && det > kSingularRel * t3 * t3 * t3) {
      const double bx = -q[3], by = -q[6], bz = -q[8];
      v = make_double3((c00 * bx + c01 * by + c02 * bz) / det, (c01 * bx + c11 * by + c12 * bz) / det,
                       (c02 * bx + c12 * by + c22 * bz) / det);
      c = qeval(q, v);
    } else {
      const double3 pm = make_double3(0.5 * (pa.x + pb.x), 0.5 * (pa.y + pb.y), 0.5 * (pa.z + pb.z));
      const double ca = qeval(q, pa), cb = qeval(q, pb), cm = qeval(q, pm);
      v = pa;
      c = ca;
      if (cb < c) { v = pb; c = cb; }
      if (cm < c) { v = pm; c = cm; }
    }
    c = fmax(c, 0.0);
    vstar[3 * e] = v.x;
    vstar[3 * e + 1] = v.y;
    vstar[3 * e + 2] = v.z;
    cost[e] = c;
    bool ok = !fixed[a] && !fixed[b];
    // link condition and the opposite vertices' degrees
    if (ok) {
      long long i = nbr_off[a], j = nbr_off[b], common = 0;
      const long long ie = nbr_off[a + 1], je = nbr_off[b + 1];
      while (i < ie && j < je && ok) {
        if (nbr[i] < nbr[j]) ++i;
        else if (nbr[j] < nbr[i]) ++j;
        else {
          const long long o = nbr[i];
          ok = nbr_off[o + 1] - nbr_off[o] >= 4;
          ++common; ++i; ++j;
        }
      }
      ok = ok && common == 2;
    }
    // no surviving face around a or b flips (turns by >= 90 degrees) or collapses to zero area
    if (ok) {
      const double3 vf32 = make_double3((double)(float)v.x, (double)(float)v.y, (double)(float)v.z);
      for (int s = 0; s < 2 && ok; ++s) {
        const long long w = s ? b : a;
        for (long long i = vf_off[w]; i < vf_off[w + 1] && ok; ++i) {
          const long long* f = faces + 3 * vf[i];
          if (has(f, a) && has(f, b)) continue;
          double3 p[3], r[3];
          for (int k = 0; k < 3; ++k) {
            p[k] = ld3(verts, f[k]);
            r[k] = f[k] == w ? vf32 : p[k];
          }
          const double3 n0 = cross(sub(p[1], p[0]), sub(p[2], p[0]));
          const double3 n1 = cross(sub(r[1], r[0]), sub(r[2], r[0]));
          ok = dot(n1, n1) > 0.0 && (dot(n0, n0) == 0.0 || dot(n0, n1) > 0.0);
        }
      }
    }
    key[e] = ok ? ((unsigned long long)__float_as_uint((float)c) << 32) | (unsigned long long)e : kNoKey;
  }
}

__global__ void __launch_bounds__(kThreads)
vertex_min_kernel(const long long* __restrict__ edges, long long E, const unsigned long long* __restrict__ key,
                  unsigned long long* __restrict__ m1) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = key[e];
    if (k == kNoKey) continue;
    atomicMin(&m1[edges[2 * e]], k);
    atomicMin(&m1[edges[2 * e + 1]], k);
  }
}

__global__ void __launch_bounds__(kThreads)
ring_min_kernel(long long V, const long long* __restrict__ nbr_off, const long long* __restrict__ nbr,
                const unsigned long long* __restrict__ m1, unsigned long long* __restrict__ m2) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    unsigned long long m = m1[v];
    for (long long j = nbr_off[v]; j < nbr_off[v + 1]; ++j) m = min(m, m1[nbr[j]]);
    m2[v] = m;
  }
}

__global__ void __launch_bounds__(kThreads)
select_kernel(const long long* __restrict__ edges, long long E, const unsigned long long* __restrict__ key,
              const unsigned long long* __restrict__ m2, uint8_t* __restrict__ sel) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = key[e];
    sel[e] = k != kNoKey && k == m2[edges[2 * e]] && k == m2[edges[2 * e + 1]];
  }
}

__global__ void __launch_bounds__(kThreads)
remap_init_kernel(const float* __restrict__ verts, long long V, long long* __restrict__ remap, float* __restrict__ pos) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    remap[v] = v;
    pos[3 * v] = verts[3 * v];
    pos[3 * v + 1] = verts[3 * v + 1];
    pos[3 * v + 2] = verts[3 * v + 2];
  }
}

__global__ void __launch_bounds__(kThreads)
collapse_edges_kernel(const long long* __restrict__ edges, long long E, const uint8_t* __restrict__ sel,
                      const double* __restrict__ vstar, long long* __restrict__ remap, float* __restrict__ pos) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    if (!sel[e]) continue;
    const long long a = edges[2 * e], b = edges[2 * e + 1];
    remap[b] = a;
    pos[3 * a] = (float)vstar[3 * e];
    pos[3 * a + 1] = (float)vstar[3 * e + 1];
    pos[3 * a + 2] = (float)vstar[3 * e + 2];
  }
}

__global__ void __launch_bounds__(kThreads)
alive_kernel(const long long* __restrict__ faces, long long V, long long F, const long long* __restrict__ remap,
             uint8_t* __restrict__ face_alive, uint8_t* __restrict__ vert_alive) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < V + F;
       t += (long long)gridDim.x * blockDim.x) {
    if (t < V) {
      vert_alive[t] = remap[t] == t;
    } else {
      const long long* f = faces + 3 * (t - V);
      const long long r0 = remap[f[0]], r1 = remap[f[1]], r2 = remap[f[2]];
      face_alive[t - V] = r0 != r1 && r1 != r2 && r0 != r2;
    }
  }
}

__global__ void __launch_bounds__(kThreads)
compact_kernel(const long long* __restrict__ faces, long long V, long long F, const long long* __restrict__ remap,
               const float* __restrict__ pos, const uint8_t* __restrict__ face_alive,
               const uint8_t* __restrict__ vert_alive, const long long* __restrict__ face_cum,
               const long long* __restrict__ vert_cum, float* __restrict__ out_verts, long long* __restrict__ out_faces) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < V + F;
       t += (long long)gridDim.x * blockDim.x) {
    if (t < V) {
      if (!vert_alive[t]) continue;
      const long long o = vert_cum[t] - 1;
      out_verts[3 * o] = pos[3 * t];
      out_verts[3 * o + 1] = pos[3 * t + 1];
      out_verts[3 * o + 2] = pos[3 * t + 2];
    } else {
      const long long f = t - V;
      if (!face_alive[f]) continue;
      const long long o = face_cum[f] - 1;
      for (int k = 0; k < 3; ++k) out_faces[3 * o + k] = vert_cum[remap[faces[3 * f + k]]] - 1;
    }
  }
}

}  // namespace

extern "C" int sr_simplify_quadrics(const float* verts, const int64_t* faces, int64_t V, int64_t F,
                                    const int64_t* vf_off, const int64_t* vf, const int64_t* nbr_off,
                                    const int64_t* nbr, double* Q, uint8_t* fixed, cudaStream_t s) {
  if (!verts || !faces || !vf_off || !vf || !nbr_off || !nbr || !Q || !fixed || V <= 0 || F <= 0) return SR_EINVAL;
  quadrics_kernel<<<sr_grid_for(V, kThreads, 8), kThreads, 0, s>>>(
      verts, (const long long*)faces, V, (const long long*)vf_off, (const long long*)vf, (const long long*)nbr_off,
      (const long long*)nbr, Q, fixed);
  return sr_launch_status();
}

extern "C" int sr_simplify_edge_cost(const float* verts, const int64_t* faces, const int64_t* edges, int64_t E,
                                     const int64_t* vf_off, const int64_t* vf, const int64_t* nbr_off,
                                     const int64_t* nbr, const double* Q, const uint8_t* fixed, double* vstar,
                                     double* cost, uint64_t* key, cudaStream_t s) {
  if (!verts || !faces || !edges || !vf_off || !vf || !nbr_off || !nbr || !Q || !fixed || !vstar || !cost || !key ||
      E <= 0 || E > 0xffffffffLL)
    return SR_EINVAL;
  edge_cost_kernel<<<sr_grid_for(E, kThreads, 8), kThreads, 0, s>>>(
      verts, (const long long*)faces, (const long long*)edges, E, (const long long*)vf_off, (const long long*)vf,
      (const long long*)nbr_off, (const long long*)nbr, Q, fixed, vstar, cost, (unsigned long long*)key);
  return sr_launch_status();
}

extern "C" int sr_simplify_select(const int64_t* edges, int64_t E, int64_t V, const int64_t* nbr_off,
                                  const int64_t* nbr, const uint64_t* key, uint64_t* m1, uint64_t* m2, uint8_t* sel,
                                  cudaStream_t s) {
  if (!edges || !nbr_off || !nbr || !key || !m1 || !m2 || !sel || E <= 0 || V <= 0) return SR_EINVAL;
  cudaError_t err = cudaMemsetAsync(m1, 0xff, (size_t)V * 8, s);
  if (err != cudaSuccess) return (int)err;
  vertex_min_kernel<<<sr_grid_for(E, kThreads, 8), kThreads, 0, s>>>(
      (const long long*)edges, E, (const unsigned long long*)key, (unsigned long long*)m1);
  ring_min_kernel<<<sr_grid_for(V, kThreads, 8), kThreads, 0, s>>>(
      V, (const long long*)nbr_off, (const long long*)nbr, (const unsigned long long*)m1, (unsigned long long*)m2);
  select_kernel<<<sr_grid_for(E, kThreads, 8), kThreads, 0, s>>>(
      (const long long*)edges, E, (const unsigned long long*)key, (const unsigned long long*)m2, sel);
  return sr_launch_status();
}

extern "C" int sr_simplify_collapse(const float* verts, const int64_t* faces, int64_t V, int64_t F,
                                    const int64_t* edges, int64_t E, const uint8_t* sel, const double* vstar,
                                    int64_t* remap, float* pos, uint8_t* face_alive, uint8_t* vert_alive,
                                    cudaStream_t s) {
  if (!verts || !faces || !edges || !sel || !vstar || !remap || !pos || !face_alive || !vert_alive || V <= 0 ||
      F <= 0 || E <= 0)
    return SR_EINVAL;
  remap_init_kernel<<<sr_grid_for(V, kThreads, 8), kThreads, 0, s>>>(verts, V, (long long*)remap, pos);
  collapse_edges_kernel<<<sr_grid_for(E, kThreads, 8), kThreads, 0, s>>>((const long long*)edges, E, sel, vstar,
                                                                         (long long*)remap, pos);
  alive_kernel<<<sr_grid_for(V + F, kThreads, 8), kThreads, 0, s>>>((const long long*)faces, V, F,
                                                                    (const long long*)remap, face_alive, vert_alive);
  return sr_launch_status();
}

extern "C" int sr_simplify_compact(const int64_t* faces, int64_t V, int64_t F, const int64_t* remap, const float* pos,
                                   const uint8_t* face_alive, const uint8_t* vert_alive, const int64_t* face_cum,
                                   const int64_t* vert_cum, float* out_verts, int64_t* out_faces, cudaStream_t s) {
  if (!faces || !remap || !pos || !face_alive || !vert_alive || !face_cum || !vert_cum || !out_verts || !out_faces ||
      V <= 0 || F <= 0)
    return SR_EINVAL;
  compact_kernel<<<sr_grid_for(V + F, kThreads, 8), kThreads, 0, s>>>(
      (const long long*)faces, V, F, (const long long*)remap, pos, face_alive, vert_alive, (const long long*)face_cum,
      (const long long*)vert_cum, out_verts, (long long*)out_faces);
  return sr_launch_status();
}
