// Pointwise stages of the tensor-core tracer (OptimizeSurfacePs, utils/FindSurfacePs.py:114-163).
// The dense layers run as wgmma split-BF16 GEMM launches (tc_gemm.cu); between them two small
// kernels do everything that is per-ray:
//   trace_mid    after the forward sweeps: LBS of p + offset (warp per ray), convergence test,
//                loss, and the cotangents that seed the two backward sweeps
//   trace_update after the backward sweeps: chain rule through the positional encodings,
//                damped Newton step p <- p - loss/|g|^2 g, device-side append to the next list
#include "common.cuh"
#include "lbs.cuh"
#include "trace_rules.cuh"

namespace {

struct MidArgs {
  const int* index;        // active list (or null = identity)
  const int* m_dev;        // device-side count (or null -> P)
  long long P;
  const float* pts;        // [P,3] canonical points (global indexing)
  const float* rays;       // [P,3]
  const long long* batch_inds;
  const float* f;          // [M] sdf value of active row i
  const float* off;        // [M][3] translator offset (or null: identity deformer)
  sr_lbs_params lbs;
  int has_lbs;
  sr_trace_params tp;
  int do_update;
  unsigned char* converged;  // [P]
  float* dsdf;             // [M][ld] cotangent rows for the SDF backward sweep (col 0)
  float* ddef;             // [M][ld] cotangent rows for the translator backward sweep (cols 0..2)
  int ld;
  float* aux;              // [M][8]: loss, state, u[3]
};

__global__ void __launch_bounds__(256) trace_mid_kernel(const __grid_constant__ MidArgs a) {
  long long M = a.P;
  if (a.m_dev) { const long long md = *a.m_dev; M = md < M ? md : M; }
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp0; i < M; i += nwarps) {
    const long long gp = a.index ? (long long)a.index[i] : i;
    float p[3], pp[3], off[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      p[j] = a.pts[gp * 3 + j];
      if (a.off) off[j] = a.off[i * 3 + j];
      pp[j] = __fadd_rn(p[j], off[j]);
    }
    float d[3], Mm[9];
    int ci[3];
    if (a.has_lbs) {
      lbs_point(a.lbs, pp, a.batch_inds ? (int)a.batch_inds[gp] : 0, d, Mm, ci);
    } else {
#pragma unroll
      for (int j = 0; j < 3; ++j) d[j] = pp[j];
#pragma unroll
      for (int q = 0; q < 9; ++q) Mm[q] = (q % 4 == 0) ? 1.f : 0.f;
    }
    if (lane == 0) {
      const float f = a.f[i];
      const RayTest r = ray_test(f, d, a.rays + gp * 3, a.tp);
      float u[3] = {0.f, 0.f, 0.f}, loss = 0.f;
      int state = 0;
      if (r.done) {
        a.converged[gp] = 1;
      } else if (a.do_update) {
        state = 1;
        loss = ray_loss(r, f, Mm, a.tp, u);
      }
      float* ax = a.aux + i * 8;
      ax[0] = loss; ax[1] = __int_as_float(state); ax[2] = u[0]; ax[3] = u[1]; ax[4] = u[2];
    }
    // cotangent rows (the whole warp writes the ld-wide rows, zero padded)
    __syncwarp();  // lane 0's aux row is visible to the whole warp
    const float* ax = a.aux + i * 8;
    for (int k = lane; k < a.ld; k += 32) {
      float vs = 0.f, vd = 0.f;
      if (k == 0) {
        const float f = a.f[i];
        vs = (__float_as_int(ax[1]) == 1) ? sdf_cotangent(f, a.tp) : 0.f;
      }
      if (k < 3) vd = ax[2 + k];
      a.dsdf[i * a.ld + k] = vs;
      if (a.ddef) a.ddef[i * a.ld + k] = vd;
    }
  }
}

struct UpdArgs {
  const int* index;
  const int* m_dev;
  long long P;
  float* pts;
  const float* gs;     // [M][gs_ld] dL/d(embedded sdf input), first 3+6L columns
  int gs_ld;
  const float* gskip;  // [M][gk_ld] skip-connection part (or null)
  int gk_ld;
  const float* gd;     // [M][gd_ld] dL/d(embedded translator input) (or null)
  int gd_ld;
  const float* aux;    // [M][8]
  int mr_s;
  float pw_s[16];
  int mr_d;
  float pw_d[16];
  int* active_out;
  int* counter_out;
};

__device__ __forceinline__ void pe_chain(const float* g, const float* gk, const float x[3], int multires,
                                         const float* pw, float out[3]) {
#pragma unroll
  for (int j = 0; j < 3; ++j) out[j] += g[j] + (gk ? gk[j] : 0.f);
  float freq = 1.0f;
  for (int b = 0; b < multires; ++b, freq *= 2.0f) {
    const float w = pw[b] * freq;
    const int ks = 3 + 6 * b, kc = ks + 3;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float sn, cs;
      sincosf(x[j] * freq, &sn, &cs);
      const float gsn = g[ks + j] + (gk ? gk[ks + j] : 0.f), gcs = g[kc + j] + (gk ? gk[kc + j] : 0.f);
      out[j] += w * (cs * gsn - sn * gcs);
    }
  }
}

__global__ void __launch_bounds__(256) trace_update_kernel(const __grid_constant__ UpdArgs a) {
  long long M = a.P;
  if (a.m_dev) { const long long md = *a.m_dev; M = md < M ? md : M; }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M;
       i += (long long)gridDim.x * blockDim.x) {
    const float* ax = a.aux + i * 8;
    if (__float_as_int(ax[1]) != 1) continue;
    const long long gp = a.index ? (long long)a.index[i] : i;
    const float x[3] = {a.pts[gp * 3], a.pts[gp * 3 + 1], a.pts[gp * 3 + 2]};
    float g[3] = {ax[2], ax[3], ax[4]};  // direct term u (d p' / d p = I + d off / d p)
    pe_chain(a.gs + i * a.gs_ld, a.gskip ? a.gskip + i * a.gk_ld : nullptr, x, a.mr_s, a.pw_s, g);
    if (a.gd) pe_chain(a.gd + i * a.gd_ld, nullptr, x, a.mr_d, a.pw_d, g);
    newton_step(a.pts + gp * 3, x, g, ax[0], a.counter_out, a.active_out, (int)gp);
  }
}

// ---- shading geometry from the tensor-core engine's outputs (infer path, network.py:356-361;
//      utils/utils.py:155-169): one warp per ray.
struct ShadePtArgs {
  long long P;
  const float* pts;
  const float* rays;
  const long long* batch_inds;
  const float* grad;   // [P][3] grad f
  const float* off4;   // [P*4][3] translator offset (row 4p) and its tangents (rows 4p+1..3), or null
  sr_lbs_params lbs;
  int has_lbs;
  float* normals;
  float* crays;
  float* dpos;
  unsigned char* inv_ok;
  float* defn;         // [P][3] deformed normal (DEFORMED instantiation only)
  float R0[9];         // camera rotation applied to defn when has_R (row-major)
  int has_R;
};

// DEFORMED also writes the deformed-surface normal normalize(J^-T g) (fallback normalize(J g) where J is singular,
// utils/utils.py:139-152) from the grad f and J the cardinal ray already uses; the other outputs are the same code.
template <bool DEFORMED>
__global__ void __launch_bounds__(256) shade_point_kernel(const __grid_constant__ ShadePtArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp0; i < a.P; i += nwarps) {
    float p[3], pp[3], off[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      p[j] = a.pts[i * 3 + j];
      if (a.off4) off[j] = a.off4[(i * 4) * 3 + j];
      pp[j] = __fadd_rn(p[j], off[j]);
    }
    float d[3], Mm[9];
    int ci[3];
    if (a.has_lbs) lbs_point(a.lbs, pp, a.batch_inds ? (int)a.batch_inds[i] : 0, d, Mm, ci);
    else {
#pragma unroll
      for (int j = 0; j < 3; ++j) d[j] = pp[j];
#pragma unroll
      for (int q = 0; q < 9; ++q) Mm[q] = (q % 4 == 0) ? 1.f : 0.f;
    }
    if (lane == 0) {
      // J = M (I + Joff), Joff[m][c] = d off_m / d p_c = off4[4i+1+c][m]
      float Q[9], m[9];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) Q[3 * r + c] = (r == c ? 1.f : 0.f) + (a.off4 ? a.off4[(i * 4 + 1 + c) * 3 + r] : 0.f);
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) m[3 * r + c] = Mm[3 * r] * Q[c] + Mm[3 * r + 1] * Q[3 + c] + Mm[3 * r + 2] * Q[6 + c];
      const bool ok = shade_point(a.grad + i * 3, m, a.rays + i * 3, a.normals + i * 3, a.crays + i * 3);
      if (a.dpos) { a.dpos[i * 3] = d[0]; a.dpos[i * 3 + 1] = d[1]; a.dpos[i * 3 + 2] = d[2]; }
      if (a.inv_ok) a.inv_ok[i] = ok ? 1 : 0;
      if constexpr (DEFORMED) {
        const float g[3] = {a.grad[i * 3], a.grad[i * 3 + 1], a.grad[i * 3 + 2]};
        float c[9], det, n[3];
        if (minv3x3_cofactors(m, c, det)) {
          // (J^-1)^T g with J^-1[r][k] = c[3k+r] / det, as shade_point applies J^-1 to v
#pragma unroll
          for (int r = 0; r < 3; ++r) n[r] = (c[3 * r] / det) * g[0] + (c[3 * r + 1] / det) * g[1] + (c[3 * r + 2] / det) * g[2];
        } else {
#pragma unroll
          for (int r = 0; r < 3; ++r) n[r] = m[3 * r] * g[0] + m[3 * r + 1] * g[1] + m[3 * r + 2] * g[2];
        }
        const float nn = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
        n[0] /= nn; n[1] /= nn; n[2] /= nn;
        if (a.has_R) {
          // diag(-1, 1, -1) R0^T n: the image's normal (model/network.py:424)
          float t[3];
#pragma unroll
          for (int r = 0; r < 3; ++r) t[r] = a.R0[r] * n[0] + a.R0[3 + r] * n[1] + a.R0[6 + r] * n[2];
          n[0] = -t[0]; n[1] = t[1]; n[2] = -t[2];
        }
        a.defn[i * 3] = n[0]; a.defn[i * 3 + 1] = n[1]; a.defn[i * 3 + 2] = n[2];
      }
    }
  }
}

// rendering_input = cat([points, PE(view_dirs), normals, feature_vectors]) (RenderNet.py:73-74)
struct RenderEmbedArgs {
  long long P;
  const float* pts;
  const float* views;
  const float* normals;
  const float* feat;   // [P][feat_ld], first nfeat columns used (starting at feat_col0)
  int feat_ld, feat_col0, nfeat, feat_row_stride;
  int multires;
  float pw[16];
  float* out;
  int ld;
};
__global__ void render_embed_kernel(const __grid_constant__ RenderEmbedArgs a) {
  const long long total = a.P * (long long)a.ld;
  const int pe = 3 + 6 * a.multires;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(idx % a.ld);
    const long long p = idx / a.ld;
    float v = 0.f;
    if (k < 3) v = a.pts[p * 3 + k];
    else if (k < 3 + pe) {
      const int q = k - 3;
      if (q < 3) v = a.views[p * 3 + q];
      else {
        const int b = (q - 3) / 6, w6 = (q - 3) % 6, j = w6 % 3;
        float sn, cs;
        sincosf(a.views[p * 3 + j] * (float)(1 << b), &sn, &cs);
        v = a.pw[b] * (w6 >= 3 ? cs : sn);
      }
    } else if (k < 3 + pe + 3) v = a.normals[p * 3 + (k - 3 - pe)];
    else if (k < 3 + pe + 3 + a.nfeat)
      v = a.feat[(size_t)p * a.feat_row_stride * a.feat_ld + a.feat_col0 + (k - 3 - pe - 3)];
    a.out[idx] = v;
  }
}

}  // namespace

extern "C" {

int sr_tc_shade_point(int64_t P, const float* pts, const float* rays, const int64_t* batch_inds,
                      const float* grad, const float* off4, const sr_lbs_params* lbs,
                      float* normals, float* crays, float* dpos, uint8_t* inv_ok, cudaStream_t s) {
  if (P <= 0 || !pts || !rays || !grad || !normals || !crays) return SR_EINVAL;
  ShadePtArgs a;
  a.P = P; a.pts = pts; a.rays = rays; a.batch_inds = (const long long*)batch_inds; a.grad = grad;
  a.off4 = off4; a.has_lbs = lbs ? 1 : 0;
  if (lbs) a.lbs = *lbs;
  a.normals = normals; a.crays = crays; a.dpos = dpos; a.inv_ok = inv_ok;
  a.defn = nullptr; a.has_R = 0;
  shade_point_kernel<false><<<sr_grid_for(P * 32, 256, 8), 256, 0, s>>>(a);
  return sr_launch_status();
}

int sr_tc_shade_point_deformed(int64_t P, const float* pts, const float* rays, const int64_t* batch_inds,
                               const float* grad, const float* off4, const sr_lbs_params* lbs,
                               float* normals, float* crays, float* dpos, uint8_t* inv_ok, float* defnormals,
                               const float* cam_R0, cudaStream_t s) {
  if (P <= 0 || !pts || !rays || !grad || !normals || !crays || !defnormals) return SR_EINVAL;
  ShadePtArgs a;
  a.P = P; a.pts = pts; a.rays = rays; a.batch_inds = (const long long*)batch_inds; a.grad = grad;
  a.off4 = off4; a.has_lbs = lbs ? 1 : 0;
  if (lbs) a.lbs = *lbs;
  a.normals = normals; a.crays = crays; a.dpos = dpos; a.inv_ok = inv_ok;
  a.defn = defnormals; a.has_R = cam_R0 ? 1 : 0;
  for (int q = 0; q < 9; ++q) a.R0[q] = cam_R0 ? cam_R0[q] : 0.f;
  shade_point_kernel<true><<<sr_grid_for(P * 32, 256, 8), 256, 0, s>>>(a);
  return sr_launch_status();
}

int sr_tc_render_embed(int64_t P, const float* pts, const float* views, const float* normals,
                       const float* feat, int feat_ld, int feat_col0, int nfeat, int feat_row_stride,
                       int multires, const float* pw, float* out, int ld, cudaStream_t s) {
  if (P <= 0 || !pts || !views || !normals || !out || !pw || (nfeat > 0 && !feat)) return SR_EINVAL;
  if (ld < 3 + 3 + 6 * multires + 3 + nfeat) return SR_EINVAL;
  RenderEmbedArgs a;
  a.P = P; a.pts = pts; a.views = views; a.normals = normals; a.feat = feat; a.feat_ld = feat_ld;
  a.feat_col0 = feat_col0; a.nfeat = nfeat; a.feat_row_stride = feat_row_stride; a.multires = multires;
  for (int i = 0; i < 16; ++i) a.pw[i] = i < multires ? pw[i] : 0.f;
  a.out = out; a.ld = ld;
  render_embed_kernel<<<sr_grid_for(P * (long long)ld, 256, 8), 256, 0, s>>>(a);
  return sr_launch_status();
}

int sr_tc_trace_mid(const int32_t* index, const int32_t* m_dev, int64_t P, const float* pts,
                    const float* rays, const int64_t* batch_inds, const float* f, const float* off,
                    const sr_lbs_params* lbs, const sr_trace_params* tp, int do_update,
                    uint8_t* converged, float* dsdf, float* ddef, int ld, float* aux, cudaStream_t s) {
  if (!pts || !rays || !f || !tp || !converged || !dsdf || !aux || P <= 0 || ld < 8) return SR_EINVAL;
  MidArgs a;
  a.index = index; a.m_dev = m_dev; a.P = P; a.pts = pts; a.rays = rays;
  a.batch_inds = (const long long*)batch_inds; a.f = f; a.off = off;
  a.has_lbs = lbs ? 1 : 0;
  if (lbs) a.lbs = *lbs;
  a.tp = *tp; a.do_update = do_update; a.converged = converged; a.dsdf = dsdf; a.ddef = ddef; a.ld = ld;
  a.aux = aux;
  trace_mid_kernel<<<sr_grid_for(P * 32, 256, 8), 256, 0, s>>>(a);
  return sr_launch_status();
}

int sr_tc_trace_update(const int32_t* index, const int32_t* m_dev, int64_t P, float* pts,
                       const float* gs, int gs_ld, const float* gskip, int gk_ld, const float* gd,
                       int gd_ld, const float* aux, int mr_s, const float* pw_s, int mr_d,
                       const float* pw_d, int32_t* active_out, int32_t* counter_out, cudaStream_t s) {
  if (!pts || !gs || !aux || !active_out || !counter_out || !pw_s || P <= 0) return SR_EINVAL;
  UpdArgs a;
  a.index = index; a.m_dev = m_dev; a.P = P; a.pts = pts; a.gs = gs; a.gs_ld = gs_ld; a.gskip = gskip;
  a.gk_ld = gk_ld; a.gd = gd; a.gd_ld = gd_ld; a.aux = aux; a.mr_s = mr_s; a.mr_d = mr_d;
  for (int i = 0; i < 16; ++i) { a.pw_s[i] = i < mr_s ? pw_s[i] : 0.f; a.pw_d[i] = (pw_d && i < mr_d) ? pw_d[i] : 0.f; }
  a.active_out = active_out; a.counter_out = counter_out;
  trace_update_kernel<<<sr_grid_for(P, 256, 8), 256, 0, s>>>(a);
  return sr_launch_status();
}
}
