// Batched singular values of 3x3 matrices on the device, with the pieces its backward needs.
// Replaces the reference's per-step CPU round trip `torch.svd(Jacobs.cpu())` in the def_regu block
// (model/network.py:573-575; SURVEY.md section 8f-2).  One thread per matrix:
//   A = J^T J (symmetric) -> cyclic Jacobi eigen-iteration (fixed 6 sweeps, fp32 storage, the rotation
//   angles in double so the eigenvalues of a near-identity J keep ~1e-7 relative accuracy)
//   s_i = sqrt(max(lambda_i, 0)) sorted descending (torch.svd's order), V = matching right singular vectors.
// Backward of a spectral loss L(s):  dL/dJ = sum_i g_i u_i v_i^T,  u_i = J v_i / s_i, u_2 = det(U) u_0 x u_1 (valid
// for repeated singular values too: only derivatives of the VALUES are propagated; see svals3x3_bwd_kernel for
// the terms below FLT_EPSILON * s_max).  Pure HBM stream: 36 B in,
// 12 (+36) B out per matrix forward; 36 + 12 + 36 + 12 in, 36 out backward.
#include <cfloat>

#include "common.cuh"

namespace {

__device__ __forceinline__ void jacobi_rotate(double a[3][3], double v[3][3], int p, int q) {
  if (fabs(a[p][q]) < 1e-300) return;
  const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
  const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
  const double app = a[p][p], aqq = a[q][q], apq = a[p][q];
  a[p][p] = app - t * apq;
  a[q][q] = aqq + t * apq;
  a[p][q] = a[q][p] = 0.0;
  const int r = 3 - p - q;
  const double arp = a[r][p], arq = a[r][q];
  a[r][p] = a[p][r] = c * arp - s * arq;
  a[r][q] = a[q][r] = s * arp + c * arq;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double vkp = v[k][p], vkq = v[k][q];
    v[k][p] = c * vkp - s * vkq;
    v[k][q] = s * vkp + c * vkq;
  }
}

__global__ void __launch_bounds__(256)
svals3x3_kernel(const float* __restrict__ J, float* __restrict__ S, float* __restrict__ V, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float m[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) m[k] = J[i * 9 + k];
    double a[3][3], v[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        a[r][c] = (double)m[r] * m[c] + (double)m[3 + r] * m[3 + c] + (double)m[6 + r] * m[6 + c];
        v[r][c] = r == c ? 1.0 : 0.0;
      }
    for (int sweep = 0; sweep < 6; ++sweep) {
      jacobi_rotate(a, v, 0, 1);
      jacobi_rotate(a, v, 0, 2);
      jacobi_rotate(a, v, 1, 2);
    }
    double lam[3] = {a[0][0], a[1][1], a[2][2]};
    int o[3] = {0, 1, 2};
    // descending order
    if (lam[o[0]] < lam[o[1]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
    if (lam[o[1]] < lam[o[2]]) { const int t = o[1]; o[1] = o[2]; o[2] = t; }
    if (lam[o[0]] < lam[o[1]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      S[i * 3 + k] = (float)sqrt(fmax(lam[o[k]], 0.0));
      if (V != nullptr) {
#pragma unroll
        for (int r = 0; r < 3; ++r) V[i * 9 + r * 3 + k] = (float)v[r][o[k]];
      }
    }
  }
}

__global__ void __launch_bounds__(256)
svals3x3_bwd_kernel(const float* __restrict__ J, const float* __restrict__ S, const float* __restrict__ V,
                    const float* __restrict__ gS, float* __restrict__ gJ, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float m[9], v[9], out[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) { m[k] = J[i * 9 + k]; v[k] = V[i * 9 + k]; out[k] = 0.f; }
    // u_k = J v_k / s_k carries an absolute error of about FLT_EPSILON * s_max (v_k is stored in fp32), i.e. a relative
    // error of FLT_EPSILON * s_max / s_k.  So the smallest one is taken as u_2 = det(U) (u_0 x u_1) instead, with
    // det(U) = sign(det J) det(V) (det J in double from the fp32 entries): accurate however small s_2 is, which keeps
    // def_regu's restoring term g_2 ~ log(s_2) / s_2 of a collapsing J.  u_0 and u_1 are dropped below FLT_EPSILON * s_max,
    // where they are noise (and then so is u_2).  The cut is relative: a J of any overall scale keeps its gradient.
    const float cut = FLT_EPSILON * S[i * 3];
    float uh[2][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float s = S[i * 3 + k], g = gS[i * 3 + k];
      const float vk[3] = {v[k], v[3 + k], v[6 + k]};
      float u[3];
      if (k < 2) {
        const float w = s > cut && s > 0.f ? g / s : 0.f;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const float jv = m[3 * r] * vk[0] + m[3 * r + 1] * vk[1] + m[3 * r + 2] * vk[2];
          u[r] = jv * w;
          uh[k][r] = s > cut && s > 0.f ? jv / s : 0.f;
        }
      } else {
        const double detJ = (double)m[0] * ((double)m[4] * m[8] - (double)m[5] * m[7]) -
                            (double)m[1] * ((double)m[3] * m[8] - (double)m[5] * m[6]) +
                            (double)m[2] * ((double)m[3] * m[7] - (double)m[4] * m[6]);
        const float detV = v[0] * (v[4] * v[8] - v[5] * v[7]) - v[1] * (v[3] * v[8] - v[5] * v[6]) +
                           v[2] * (v[3] * v[7] - v[4] * v[6]);
        const float sg = ((detJ < 0.0) != (detV < 0.f) ? -1.f : 1.f) * g;
        u[0] = (uh[0][1] * uh[1][2] - uh[0][2] * uh[1][1]) * sg;
        u[1] = (uh[0][2] * uh[1][0] - uh[0][0] * uh[1][2]) * sg;
        u[2] = (uh[0][0] * uh[1][1] - uh[0][1] * uh[1][0]) * sg;
      }
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) out[3 * r + c] += u[r] * vk[c];
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) gJ[i * 9 + k] = out[k];
  }
}

}  // namespace

extern "C" {

int sr_svals3x3_f32(const float* J, float* S, float* V, int64_t n, cudaStream_t s) {
  if (n < 0 || (n > 0 && (!J || !S))) return SR_EINVAL;
  if (n == 0) return SR_OK;
  svals3x3_kernel<<<sr_grid_for(n, 256, 8), 256, 0, s>>>(J, S, V, n);
  return sr_launch_status();
}

int sr_svals3x3_bwd_f32(const float* J, const float* S, const float* V, const float* gS, float* gJ, int64_t n,
                        cudaStream_t s) {
  if (n < 0 || (n > 0 && (!J || !S || !V || !gS || !gJ))) return SR_EINVAL;
  if (n == 0) return SR_OK;
  svals3x3_bwd_kernel<<<sr_grid_for(n, 256, 8), 256, 0, s>>>(J, S, V, gS, gJ, n);
  return sr_launch_status();
}
}
