// Per-ray rules of OptimizeSurfacePs (utils/FindSurfacePs.py:114-163) and of the shading geometry
// (model/network.py:356-361, utils/utils.py:155-169), shared by the fp32 tracers (mlp_kernels.cu), the
// tensor-core tracer's pointwise kernels (trace_tc.cu) and FastMinv's batched inverse (minv3x3.cu).
// Each engine evaluates f, D(p), M = dD/dp' and the gradient chain its own way; the decisions and the
// arithmetic around them are defined here once, so every engine takes them with the same rounding.
#pragma once
#include "common.cuh"

// Convergence test of one ray v at its point's deformed position D(p):
// u = D(p) - cam, up = u x v, sin = |up| / |u|, done = |f| < dthreshold && asin(sin) [degrees] < athreshold.
struct RayTest {
  float vx, vy, vz, ux, uy, uz, cx, cy, cz, n_up, n_u, sang;
  bool done;
};

__device__ __forceinline__ RayTest ray_test(float f, const float* d, const float* v, const sr_trace_params& tp) {
  RayTest r;
  r.vx = v[0]; r.vy = v[1]; r.vz = v[2];
  r.ux = d[0] - tp.cam_pos[0]; r.uy = d[1] - tp.cam_pos[1]; r.uz = d[2] - tp.cam_pos[2];
  r.cx = r.uy * r.vz - r.uz * r.vy; r.cy = r.uz * r.vx - r.ux * r.vz; r.cz = r.ux * r.vy - r.uy * r.vx;
  r.n_up = sqrtf(r.cx * r.cx + r.cy * r.cy + r.cz * r.cz);
  r.n_u = sqrtf(r.ux * r.ux + r.uy * r.uy + r.uz * r.uz);
  r.sang = r.n_up / r.n_u;
  const float ang = asinf(r.sang) * 180.0f / 3.14159265358979323846f;
  r.done = (fabsf(f) < tp.dthreshold) && (ang < tp.athreshold);
  return r;
}

// d loss / d f = w1 sign(f): the cotangent that seeds the SDF's reverse sweep
__device__ __forceinline__ float sdf_cotangent(float f, const sr_trace_params& tp) {
  return tp.w1 * (f > 0.f ? 1.f : (f < 0.f ? -1.f : 0.f));
}

// Returns loss = w1 |f| + w2 sin of a ray that failed the test, and writes u = w2 M^T q, the cotangent of
// p' = p + offset (also the direct dD/dp term), where q = d sin / d u (zero when up = 0) and M = dD/dp'.
// The forward-mode tracer passes J = dD/dp for M, so that u is its whole translator term.
__device__ __forceinline__ float ray_loss(const RayTest& r, float f, const float* M, const sr_trace_params& tp,
                                          float u[3]) {
  const float loss = tp.w1 * fabsf(f) + tp.w2 * fabsf(r.sang);
  float q[3] = {0.f, 0.f, 0.f};
  if (r.n_up > 0.f) {
    // d n_up / d u = (v x up) / n_up
    const float wx = r.vy * r.cz - r.vz * r.cy, wy = r.vz * r.cx - r.vx * r.cz, wz = r.vx * r.cy - r.vy * r.cx;
    const float i1 = 1.0f / (r.n_up * r.n_u), i2 = r.n_up / (r.n_u * r.n_u * r.n_u);
    q[0] = wx * i1 - r.ux * i2; q[1] = wy * i1 - r.uy * i2; q[2] = wz * i1 - r.uz * i2;
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) u[j] = tp.w2 * (M[j] * q[0] + M[3 + j] * q[1] + M[6 + j] * q[2]);
  return loss;
}

// Damped Newton step p <- x - loss / |g|^2 g (g = d loss / d p), then ray gp joins the next active list.
__device__ __forceinline__ void newton_step(float* p, const float* x, const float g[3], float loss, int32_t* counter,
                                            int32_t* active_out, int gp) {
  const float t = -loss / (g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
#pragma unroll
  for (int j = 0; j < 3; ++j) p[j] = x[j] + t * g[j];
  const int slot = atomicAdd(counter, 1);
  active_out[slot] = gp;
}

// FastMinv's 3x3 inverse rule (FastMinv/Matrix3x3InvKernels.cu:22-104): the cofactors c[3r+k] of m and
// det = row 0 . cofactors, so that the inverse is c[3k+r] / det; m is singular (inverse 0) when |det| < 1e-4,
// compared in double.  The cofactors are written as the reference writes them, so that nvcc's FMA contraction
// rounds them the same way.  det is accumulated with explicit FMAs: left to contraction, its rounding would
// depend on the calling kernel.  Returns whether m is invertible.
template <typename T>
__device__ __forceinline__ bool minv3x3_cofactors(const T* m, T c[9], T& det) {
  c[0] = m[4] * m[8] - m[5] * m[7]; c[1] = -m[3] * m[8] + m[5] * m[6]; c[2] = m[3] * m[7] - m[4] * m[6];
  c[3] = -m[1] * m[8] + m[2] * m[7]; c[4] = m[0] * m[8] - m[2] * m[6]; c[5] = -m[0] * m[7] + m[1] * m[6];
  c[6] = m[1] * m[5] - m[2] * m[4]; c[7] = -m[0] * m[5] + m[2] * m[3]; c[8] = m[0] * m[4] - m[1] * m[3];
  det = fma(m[2], c[2], fma(m[1], c[1], m[0] * c[0]));
  return !(fabs((double)det) < 0.0001);
}

// Shading geometry of one surface point: normal = normalize(grad f), cardinal ray = normalize(J^-1 v), with v in
// place of J^-1 v when J is singular.  Returns whether J was inverted.
__device__ __forceinline__ bool shade_point(const float* grad, const float* J, const float* v, float* normal,
                                            float* cray) {
  const float gx = grad[0], gy = grad[1], gz = grad[2];
  const float gn = sqrtf(gx * gx + gy * gy + gz * gz);
  normal[0] = gx / gn; normal[1] = gy / gn; normal[2] = gz / gn;
  float c[9], det;
  const bool ok = minv3x3_cofactors(J, c, det);
  const float vx = v[0], vy = v[1], vz = v[2];
  float rx = vx, ry = vy, rz = vz;
  if (ok) {
    rx = (c[0] / det) * vx + (c[3] / det) * vy + (c[6] / det) * vz;
    ry = (c[1] / det) * vx + (c[4] / det) * vy + (c[7] / det) * vz;
    rz = (c[2] / det) * vx + (c[5] / det) * vy + (c[8] / det) * vz;
  }
  const float rn = sqrtf(rx * rx + ry * ry + rz * rz);
  cray[0] = rx / rn; cray[1] = ry / rn; cray[2] = rz / rn;
  return ok;
}
