// Template mesh regularisers of OptimNetwork.computeTmpPcLoss (model/network.py:655-670): pytorch3d 0.4.0's
// mesh_laplacian_smoothing(method='uniform'), mesh_edge_loss(target_length=0.) and mesh_normal_consistency of one mesh,
// forward and backward w.r.t. the vertices.
//
// Topology (Meshes._compute_packed, once per face table).  Entry 3f+k is the edge opposite corner k of face f, sorted so
// that a <= b, with the hash V*a + b.  A stable sort of the hashes (by the caller) lists the unique edges in ascending
// hash order and, inside each edge, its (face, corner) entries in ascending order.  sr_mesh_reg_edge_runs marks the head
// of each run and its pair count; after the caller's prefix sums, sr_mesh_reg_topology writes the edge list,
// face_to_edge, the directed neighbour keys and pytorch3d's literal pair list of mesh_normal_consistency:
//   [e[i], e[j]] for i in range(m-1) for j in range(1, m) if i != j      ((m-1)^2 - (m-2) pairs for m >= 2, else 0)
// One thread per sorted entry; a run's head writes its edge and its pairs, so nothing is accumulated across threads.
//
// Forward (one grid-stride pass over V vertices + E edges + P pairs, then a one-block pass over the block partials in
// a fixed order; fp64 from the fp32 positions, as mesh_shade.cu's cross products):
//   laplacian  sum_i |(L v)_i| / V,  (L v)_i = sum_{k in N(i)} v_k / deg_i - v_i  (-v_i when deg_i = 0); N(i) is the
//              directed multiset of the unique edges (Meshes.laplacian_packed: a self-edge (a,a) counts twice)
//   edge       sum_e |v_a - v_b|^2 / E
//   normal     sum_p (1 - cos(n_i, -n_j)) / P (0 when P = 0), n = (v_b - v_a) x (v_o - v_a) for the pair's edge (a,b)
//              and each entry's opposite corner o; cos = w12 / sqrt(max(w1 w2, 1e-16)) (torch 1.10 cosine_similarity).
//              n is exactly 0, with no gradient, where it vanishes for every position (o = a, o = b or a = b: a face
//              with a repeated index); pytorch3d's literal sum of three cross products leaves rounding noise there
//              that the clamp's 1/eps would turn into a meaningless gradient.
// It keeps u_i = (L v)_i / |(L v)_i| (0 at a zero norm) and each pair's d(1 - cos)/dn_i, d/dn_j for the backward.
// Backward: one thread per vertex j gathers, in CSR order, with no atomics (bit-identical reruns):
//   (g_lap / V) (-u_j + sum_{i in N(j)} u_i / deg_i) + (2 g_edge / E) sum_{k in N(j)} (v_j - v_k)
//   + (g_norm / P) sum over the (pair, role) entries of j of the chain of d/dn through n = e1 x e2.
// All three terms are gathers over short lists (a vertex has ~6 neighbours and ~12 pair entries on a closed
// marching-cubes surface): latency / L2 bound, the positions are read a few times each from L2.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr double kEps2 = 1e-16;   // cosine_similarity's eps^2, eps = 1e-8

__global__ void __launch_bounds__(kThreads)
edge_keys_kernel(const long long* __restrict__ faces, long long F, long long V, long long* __restrict__ keys) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < 3 * F;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long f = idx / 3, k = idx % 3;
    const long long a = faces[f * 3 + (k + 1) % 3], b = faces[f * 3 + (k + 2) % 3];
    if (a < 0 || a >= V || b < 0 || b >= V)
      keys[idx] = -1;
    else
      keys[idx] = a < b ? V * a + b : V * b + a;
  }
}

__device__ __forceinline__ long long run_length(const long long* __restrict__ skeys, long long n, long long i) {
  long long m = 1;
  while (i + m < n && skeys[i + m] == skeys[i]) ++m;
  return m;
}

__device__ __forceinline__ long long pair_count(long long m) { return m < 2 ? 0 : (m - 1) * (m - 1) - (m - 2); }

__global__ void __launch_bounds__(kThreads)
edge_runs_kernel(const long long* __restrict__ skeys, long long n, long long* __restrict__ head,
                 long long* __restrict__ npairs) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const bool h = i == 0 || skeys[i] != skeys[i - 1];
    head[i] = h;
    npairs[i] = h ? pair_count(run_length(skeys, n, i)) : 0;
  }
}

__global__ void __launch_bounds__(kThreads)
topology_kernel(const long long* __restrict__ faces, const long long* __restrict__ skeys,
                const long long* __restrict__ perm, const long long* __restrict__ head_cum,
                const long long* __restrict__ pair_cum, long long n, long long V, long long* __restrict__ edges,
                long long* __restrict__ face_to_edge, long long* __restrict__ dir_keys, long long* __restrict__ pairs) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long e = head_cum[i] - 1;
    face_to_edge[perm[i]] = e;
    if (i != 0 && skeys[i] == skeys[i - 1]) continue;
    const long long key = skeys[i], a = key / V, b = key % V;
    edges[2 * e] = a;
    edges[2 * e + 1] = b;
    dir_keys[2 * e] = V * a + b;
    dir_keys[2 * e + 1] = V * b + a;
    const long long m = run_length(skeys, n, i);
    long long p = i == 0 ? 0 : pair_cum[i - 1];
    for (long long x = 0; x < m - 1; ++x)
      for (long long y = 1; y < m; ++y) {
        if (x == y) continue;
        // perm holds the entry ids 3f+k: the corner opposite the edge is faces[3f+k]
        pairs[4 * p] = a;
        pairs[4 * p + 1] = b;
        pairs[4 * p + 2] = faces[perm[i + x]];
        pairs[4 * p + 3] = faces[perm[i + y]];
        ++p;
      }
  }
}

__device__ __forceinline__ double3 ld3(const float* __restrict__ v, long long i) {
  return make_double3((double)v[3 * i], (double)v[3 * i + 1], (double)v[3 * i + 2]);
}
__device__ __forceinline__ double3 sub(double3 a, double3 b) { return make_double3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double dot(double3 a, double3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ double3 cross(double3 a, double3 b) {
  return make_double3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ void acc(double3& s, double3 a) { s.x += a.x; s.y += a.y; s.z += a.z; }

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sums three values over the block in a fixed order; thread 0 gets the result.
__device__ __forceinline__ void block_sum3(double v[3]) {
  __shared__ double red[3][kThreads / 32];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    v[c] = warp_sum_d(v[c]);
    if (l == 0) red[c][w] = v[c];
  }
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double s = 0.0;
      for (int k = 0; k < kThreads / 32; ++k) s += red[c][k];
      v[c] = s;
    }
}

__global__ void __launch_bounds__(kThreads)
forward_kernel(const float* __restrict__ verts, long long V, long long E, long long P, const long long* __restrict__ edges,
               const long long* __restrict__ nbr_off, const long long* __restrict__ nbr,
               const long long* __restrict__ pairs, double* __restrict__ u, double* __restrict__ dn,
               double* __restrict__ partials) {
  double s[3] = {0.0, 0.0, 0.0};   // laplacian, edge, normal consistency
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < V + E + P;
       t += (long long)gridDim.x * blockDim.x) {
    if (t < V) {
      const long long k0 = nbr_off[t], k1 = nbr_off[t + 1];
      double3 sum = make_double3(0.0, 0.0, 0.0);
      for (long long k = k0; k < k1; ++k) acc(sum, ld3(verts, nbr[k]));
      const double inv = k1 > k0 ? 1.0 / (double)(k1 - k0) : 0.0;
      const double3 vi = ld3(verts, t);
      const double3 lv = make_double3(sum.x * inv - vi.x, sum.y * inv - vi.y, sum.z * inv - vi.z);
      const double nrm = sqrt(dot(lv, lv));
      s[0] += nrm;
      const double r = nrm > 0.0 ? 1.0 / nrm : 0.0;
      u[3 * t] = lv.x * r;
      u[3 * t + 1] = lv.y * r;
      u[3 * t + 2] = lv.z * r;
    } else if (t < V + E) {
      const long long e = t - V;
      const double3 d = sub(ld3(verts, edges[2 * e]), ld3(verts, edges[2 * e + 1]));
      s[1] += dot(d, d);
    } else {
      const long long p = t - V - E;
      const long long a = pairs[4 * p], b = pairs[4 * p + 1], oi = pairs[4 * p + 2], oj = pairs[4 * p + 3];
      // a normal that is zero for every position (corner on the edge, or a self-edge) is exactly 0, with no gradient
      const bool zi = a == b || oi == a || oi == b, zj = a == b || oj == a || oj == b;
      const double3 va = ld3(verts, a), e1 = sub(ld3(verts, b), va), zero = make_double3(0.0, 0.0, 0.0);
      const double3 ni = zi ? zero : cross(e1, sub(ld3(verts, oi), va));
      const double3 nj = zj ? zero : cross(e1, sub(ld3(verts, oj), va));
      // 1 - cos(n_i, -n_j) = 1 + d / sq, sq = sqrt(max(w1 w2, eps^2)); below the clamp sq is constant
      const double d = dot(ni, nj), w1 = dot(ni, ni), w2 = dot(nj, nj), q = w1 * w2;
      const bool live = q >= kEps2;
      const double sq = sqrt(live ? q : kEps2), isq = 1.0 / sq;
      s[2] += 1.0 + d * isq;
      const double ci = live ? d * w2 / q : 0.0, cj = live ? d * w1 / q : 0.0;
      const double si = zi ? 0.0 : isq, sj = zj ? 0.0 : isq;
      double* o = dn + 6 * p;
      o[0] = (nj.x - ci * ni.x) * si;
      o[1] = (nj.y - ci * ni.y) * si;
      o[2] = (nj.z - ci * ni.z) * si;
      o[3] = (ni.x - cj * nj.x) * sj;
      o[4] = (ni.y - cj * nj.y) * sj;
      o[5] = (ni.z - cj * nj.z) * sj;
    }
  }
  block_sum3(s);
  if (threadIdx.x == 0) {
    partials[3 * blockIdx.x] = s[0];
    partials[3 * blockIdx.x + 1] = s[1];
    partials[3 * blockIdx.x + 2] = s[2];
  }
}

__global__ void __launch_bounds__(kThreads)
finish_kernel(const double* __restrict__ partials, int nblocks, long long V, long long E, long long P,
              float* __restrict__ out) {
  double s[3] = {0.0, 0.0, 0.0};
  for (int b = threadIdx.x; b < nblocks; b += kThreads) {
    s[0] += partials[3 * b];
    s[1] += partials[3 * b + 1];
    s[2] += partials[3 * b + 2];
  }
  block_sum3(s);
  if (threadIdx.x == 0) {
    out[0] = (float)(s[0] / (double)V);
    out[1] = (float)(s[1] / (double)E);
    out[2] = P > 0 ? (float)(s[2] / (double)P) : 0.f;
  }
}

__global__ void __launch_bounds__(kThreads)
backward_kernel(const float* __restrict__ verts, long long V, long long E, long long P,
                const long long* __restrict__ nbr_off, const long long* __restrict__ nbr,
                const long long* __restrict__ pairs, const long long* __restrict__ vp_off,
                const long long* __restrict__ vp_ent, const double* __restrict__ u, const double* __restrict__ dn,
                const float* __restrict__ grad_out, float* __restrict__ grad_verts) {
  const double cl = (double)grad_out[0] / (double)V, ce = 2.0 * (double)grad_out[1] / (double)E,
               cn = P > 0 ? (double)grad_out[2] / (double)P : 0.0;
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < V; j += (long long)gridDim.x * blockDim.x) {
    const double3 vj = ld3(verts, j);
    double3 gl = make_double3(0.0, 0.0, 0.0), ge = gl, gn = gl;
    for (long long k = nbr_off[j]; k < nbr_off[j + 1]; ++k) {
      const long long i = nbr[k];
      const double inv = 1.0 / (double)(nbr_off[i + 1] - nbr_off[i]);   // deg_i >= 1: j is a neighbour of i
      gl.x += u[3 * i] * inv;
      gl.y += u[3 * i + 1] * inv;
      gl.z += u[3 * i + 2] * inv;
      acc(ge, sub(vj, ld3(verts, i)));
    }
    for (long long r = vp_off[j]; r < vp_off[j + 1]; ++r) {
      const long long ent = vp_ent[r], p = ent >> 2;
      const int role = (int)(ent & 3);
      const double* g = dn + 6 * p;
      const double3 gi = make_double3(g[0], g[1], g[2]), gj = make_double3(g[3], g[4], g[5]);
      const double3 va = ld3(verts, pairs[4 * p]), vb = ld3(verts, pairs[4 * p + 1]);
      // n = e1 x e2, e1 = v_b - v_a, e2 = v_o - v_a:  dn/dv_b^T g = e2 x g, dn/dv_o^T g = g x e1,
      // dn/dv_a^T g = (v_b - v_o) x g
      if (role == 0) {
        acc(gn, cross(sub(vb, ld3(verts, pairs[4 * p + 2])), gi));
        acc(gn, cross(sub(vb, ld3(verts, pairs[4 * p + 3])), gj));
      } else if (role == 1) {
        acc(gn, cross(sub(ld3(verts, pairs[4 * p + 2]), va), gi));
        acc(gn, cross(sub(ld3(verts, pairs[4 * p + 3]), va), gj));
      } else {
        acc(gn, cross(role == 2 ? gi : gj, sub(vb, va)));
      }
    }
    const double* uj = u + 3 * j;
    grad_verts[3 * j] = (float)(cl * (gl.x - uj[0]) + ce * ge.x + cn * gn.x);
    grad_verts[3 * j + 1] = (float)(cl * (gl.y - uj[1]) + ce * ge.y + cn * gn.y);
    grad_verts[3 * j + 2] = (float)(cl * (gl.z - uj[2]) + ce * ge.z + cn * gn.z);
  }
}

// V * V must fit the int64 edge hash
constexpr long long kMaxVerts = 1LL << 31;

}  // namespace

extern "C" int sr_mesh_reg_edge_keys(const int64_t* faces, int64_t F, int64_t V, int64_t* keys, cudaStream_t s) {
  if (!faces || !keys || F <= 0 || V <= 0 || V > kMaxVerts) return SR_EINVAL;
  edge_keys_kernel<<<sr_grid_for(3 * F, kThreads, 8), kThreads, 0, s>>>((const long long*)faces, F, V,
                                                                          (long long*)keys);
  return sr_launch_status();
}

extern "C" int sr_mesh_reg_edge_runs(const int64_t* sorted_keys, int64_t n, int64_t* head, int64_t* npairs,
                                     cudaStream_t s) {
  if (!sorted_keys || !head || !npairs || n <= 0) return SR_EINVAL;
  edge_runs_kernel<<<sr_grid_for(n, kThreads, 8), kThreads, 0, s>>>((const long long*)sorted_keys, n,
                                                                      (long long*)head, (long long*)npairs);
  return sr_launch_status();
}

extern "C" int sr_mesh_reg_topology(const int64_t* faces, const int64_t* sorted_keys, const int64_t* perm,
                                    const int64_t* head_cum, const int64_t* pair_cum, int64_t F, int64_t V, int64_t E,
                                    int64_t P, int64_t* edges, int64_t* face_to_edge, int64_t* dir_keys, int64_t* pairs,
                                    cudaStream_t s) {
  if (!faces || !sorted_keys || !perm || !head_cum || !pair_cum || !edges || !face_to_edge || !dir_keys ||
      (P > 0 && !pairs) || F <= 0 || V <= 0 || V > kMaxVerts || E <= 0 || E > 3 * F || P < 0)
    return SR_EINVAL;
  topology_kernel<<<sr_grid_for(3 * F, kThreads, 8), kThreads, 0, s>>>(
      (const long long*)faces, (const long long*)sorted_keys, (const long long*)perm, (const long long*)head_cum,
      (const long long*)pair_cum, 3 * F, V, (long long*)edges, (long long*)face_to_edge, (long long*)dir_keys,
      (long long*)pairs);
  return sr_launch_status();
}

extern "C" int sr_mesh_reg_forward(const float* verts, int64_t V, int64_t E, int64_t P, const int64_t* edges,
                                   const int64_t* nbr_off, const int64_t* nbr, const int64_t* pairs, double* u,
                                   double* dn, double* partials, float* out, cudaStream_t s) {
  if (!verts || !edges || !nbr_off || !nbr || !u || !partials || !out || (P > 0 && (!pairs || !dn)) || V <= 0 ||
      E <= 0 || P < 0)
    return SR_EINVAL;
  const int grid = sr_grid_for(V + E + P, kThreads, SR_MESH_REG_BLOCKS / SR_NUM_SMS);
  forward_kernel<<<grid, kThreads, 0, s>>>(verts, V, E, P, (const long long*)edges, (const long long*)nbr_off,
                                           (const long long*)nbr, (const long long*)pairs, u, dn, partials);
  finish_kernel<<<1, kThreads, 0, s>>>(partials, grid, V, E, P, out);
  return sr_launch_status();
}

extern "C" int sr_mesh_reg_backward(const float* verts, int64_t V, int64_t E, int64_t P, const int64_t* nbr_off,
                                    const int64_t* nbr, const int64_t* pairs, const int64_t* vp_off,
                                    const int64_t* vp_ent, const double* u, const double* dn, const float* grad_out,
                                    float* grad_verts, cudaStream_t s) {
  if (!verts || !nbr_off || !nbr || !vp_off || !u || !grad_out || !grad_verts ||
      (P > 0 && (!pairs || !vp_ent || !dn)) || V <= 0 || E <= 0 || P < 0)
    return SR_EINVAL;
  backward_kernel<<<sr_grid_for(V, kThreads, 8), kThreads, 0, s>>>(
      verts, V, E, P, (const long long*)nbr_off, (const long long*)nbr, (const long long*)pairs,
      (const long long*)vp_off, (const long long*)vp_ent, u, dn, grad_out, grad_verts);
  return sr_launch_status();
}
