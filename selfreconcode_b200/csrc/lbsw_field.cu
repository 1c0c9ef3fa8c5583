// Skin-weight volume of a new sequence (the reference's compute_lbswField, model/Deformer.py:246-284 and
// utils/LBSWsmpl.py:14-52): an inverse-distance blend of the skin weights of the k nearest template vertices at every
// voxel centre, then damped 6-neighbour smoothing passes with per-voxel renormalisation.
//
// sr_lbsw_knn_blend (one thread per voxel, x fastest):
//   centre  u = i / W + (1 / W) / 2 (i / (W - 1) with align_corners), p = u * (hi - lo) + lo: the fp32 operations of
//           voxel_centres() (dropin/utils/LBSWsmpl.py) one by one with round-to-nearest intrinsics, so that nothing is
//           contracted into an FMA and the centres are bit-identical to torch's.
//   k-NN    the vertices stream through shared memory in tiles of float4; each thread keeps its k smallest
//           (d^2, index) pairs sorted in registers (an unrolled insertion).  Candidates come in index order and only a
//           strictly smaller d^2 enters, so equal distances keep the lower index.
//   blend   w_n = 1 / min(max(sqrt(d2_n), 1e-4), 1), normalised by their sum (ascending order), field[c] =
//           sum_n w_n ws[idx_n, c] in ascending distance order.
// sr_lbsw_smooth_pass (one thread per voxel, src -> dst: a Jacobi pass):  interior voxels take (c - mean) * 0.7 + mean
//   with mean = (+z + -z + +y + -y + +x + -x) / 6 of src (the reference's order), boundary voxels keep theirs; every
//   voxel is then divided by its channel sum and, with cut > 0, values below cut become 0.
// No atomics: reruns are bit-identical.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kBlendThreads = 128;
constexpr int kTile = 1024;          // vertices per shared-memory tile (16 KB)
constexpr int kSmoothThreads = 256;

__device__ __forceinline__ float voxel_coord(int i, int n, float lo, float hi, int align) {
  const float fi = (float)i, fn = (float)n;
  const float u = align ? __fdiv_rn(fi, __fsub_rn(fn, 1.f))
                        : __fadd_rn(__fdiv_rn(fi, fn), __fmul_rn(__fdiv_rn(1.f, fn), 0.5f));
  return __fadd_rn(__fmul_rn(u, __fsub_rn(hi, lo)), lo);
}

// KM = list length in registers; kFixed: k == KM (the sizes the code uses), else k <= KM is a runtime value.
template <int KM, bool kFixed>
__global__ void __launch_bounds__(kBlendThreads)
lbsw_blend_kernel(const float* __restrict__ verts, const float* __restrict__ ws, int V, int C, float3 lo, float3 hi,
                  int W, int H, int D, int align, int k_arg, float* __restrict__ field, float* __restrict__ centres) {
  __shared__ float4 tile[kTile];
  const int k = kFixed ? KM : k_arg;
  const long long n = (long long)W * H * D;
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = v < n;
  const long long vv = live ? v : 0;
  const int i = (int)(vv % W), j = (int)((vv / W) % H), l = (int)(vv / ((long long)W * H));
  const float px = voxel_coord(i, W, lo.x, hi.x, align);
  const float py = voxel_coord(j, H, lo.y, hi.y, align);
  const float pz = voxel_coord(l, D, lo.z, hi.z, align);

  // Sorted ascending; the first KM - k slots hold -inf sentinels that no candidate displaces, so the k real entries
  // are slots KM - k .. KM - 1 and the k-th smallest is always dk[KM - 1].
  const int k0 = KM - k;
  float dk[KM];
  int ik[KM];
#pragma unroll
  for (int s = 0; s < KM; ++s) {
    dk[s] = s < k0 ? -INFINITY : INFINITY;
    ik[s] = 0;
  }
  for (int t0 = 0; t0 < V; t0 += kTile) {
    const int nt = min(kTile, V - t0);
    __syncthreads();
    for (int q = threadIdx.x; q < nt; q += blockDim.x) {
      const float* p = verts + (long long)(t0 + q) * 3;
      tile[q] = make_float4(p[0], p[1], p[2], 0.f);
    }
    __syncthreads();
    if (!live) continue;
#pragma unroll 4
    for (int q = 0; q < nt; ++q) {
      const float4 c = tile[q];
      const float dx = __fsub_rn(px, c.x), dy = __fsub_rn(py, c.y), dz = __fsub_rn(pz, c.z);
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      if (d2 < dk[KM - 1]) {
        const int idx = t0 + q;
#pragma unroll
        for (int s = KM - 1; s > 0; --s) {
          if (d2 < dk[s - 1]) {
            dk[s] = dk[s - 1];
            ik[s] = ik[s - 1];
          } else if (d2 < dk[s]) {
            dk[s] = d2;
            ik[s] = idx;
          }
        }
        if (d2 < dk[0]) {
          dk[0] = d2;
          ik[0] = idx;
        }
      }
    }
  }
  if (!live) return;
  if (centres) {
    centres[v * 3] = px;
    centres[v * 3 + 1] = py;
    centres[v * 3 + 2] = pz;
  }
  float wsum = 0.f;
#pragma unroll
  for (int s = 0; s < KM; ++s) {
    if (s >= k0) {
      dk[s] = __frcp_rn(fminf(fmaxf(__fsqrt_rn(dk[s]), 1e-4f), 1.f));
      wsum = __fadd_rn(wsum, dk[s]);
    }
  }
#pragma unroll
  for (int s = 0; s < KM; ++s)
    if (s >= k0) dk[s] = __fdiv_rn(dk[s], wsum);
  for (int c = 0; c < C; ++c) {
    float acc = 0.f;
#pragma unroll
    for (int s = 0; s < KM; ++s)
      if (s >= k0) acc = __fadd_rn(acc, __fmul_rn(dk[s], __ldg(ws + (long long)ik[s] * C + c)));
    field[(long long)c * n + v] = acc;
  }
}

__global__ void __launch_bounds__(kSmoothThreads)
lbsw_smooth_kernel(const float* __restrict__ src, float* __restrict__ dst, int C, int D, int H, int W, float cut) {
  const long long HW = (long long)H * W, n = HW * D;
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(v % W), y = (int)((v / W) % H), z = (int)(v / HW);
    const bool inner = x >= 1 && x <= W - 2 && y >= 1 && y <= H - 2 && z >= 1 && z <= D - 2;
    float val[SR_LBSW_MAX_C];
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < SR_LBSW_MAX_C; ++c) {
      if (c < C) {
        const float* p = src + (long long)c * n + v;
        float a = p[0];
        if (inner) {
          float m = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(p[HW], p[-HW]), p[W]), p[-W]), p[1]), p[-1]);
          m = __fdiv_rn(m, 6.f);
          a = __fadd_rn(__fmul_rn(__fsub_rn(a, m), 0.7f), m);
        }
        val[c] = a;
        sum = __fadd_rn(sum, a);
      }
    }
#pragma unroll
    for (int c = 0; c < SR_LBSW_MAX_C; ++c) {
      if (c < C) {
        float r = __fdiv_rn(val[c], sum);
        if (cut > 0.f && r < cut) r = 0.f;
        dst[(long long)c * n + v] = r;
      }
    }
  }
}

__global__ void __launch_bounds__(256) lbsw_cut_kernel(float* __restrict__ field, long long n, float cut) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
    if (field[t] < cut) field[t] = 0.f;
}

}  // namespace

extern "C" int sr_lbsw_knn_blend(const float* verts, const float* vert_ws, int V, int C, const float* bmin,
                                 const float* bmax, int W, int H, int D, int align_corners, int k, float* field,
                                 float* centres, cudaStream_t s) {
  if (!verts || !vert_ws || !bmin || !bmax || !field || V < 1 || C < 1 || C > SR_LBSW_MAX_C || k < 1 ||
      k > SR_LBSW_MAX_K || k > V || W < 1 || H < 1 || D < 1)
    return SR_EINVAL;
  const long long n = (long long)W * H * D;
  const int blocks = sr_div_up(n, kBlendThreads);
  const float3 lo = make_float3(bmin[0], bmin[1], bmin[2]), hi = make_float3(bmax[0], bmax[1], bmax[2]);
  const int al = align_corners ? 1 : 0;
  if (k == 5)
    lbsw_blend_kernel<5, true><<<blocks, kBlendThreads, 0, s>>>(verts, vert_ws, V, C, lo, hi, W, H, D, al, k, field,
                                                                centres);
  else if (k == 30)
    lbsw_blend_kernel<30, true><<<blocks, kBlendThreads, 0, s>>>(verts, vert_ws, V, C, lo, hi, W, H, D, al, k, field,
                                                                 centres);
  else
    lbsw_blend_kernel<SR_LBSW_MAX_K, false><<<blocks, kBlendThreads, 0, s>>>(verts, vert_ws, V, C, lo, hi, W, H, D,
                                                                             al, k, field, centres);
  return sr_launch_status();
}

extern "C" int sr_lbsw_smooth_pass(const float* src, float* dst, int C, int D, int H, int W, float cut,
                                   cudaStream_t s) {
  if (!src || !dst || src == dst || C < 1 || C > SR_LBSW_MAX_C || D < 1 || H < 1 || W < 1 || !(cut >= 0.f))
    return SR_EINVAL;
  const long long n = (long long)D * H * W;
  lbsw_smooth_kernel<<<sr_grid_for(n, kSmoothThreads, 16), kSmoothThreads, 0, s>>>(src, dst, C, D, H, W, cut);
  return sr_launch_status();
}

extern "C" int sr_lbsw_cut(float* field, int64_t n, float cut, cudaStream_t s) {
  if (!field || n < 1 || !(cut >= 0.f)) return SR_EINVAL;
  lbsw_cut_kernel<<<sr_grid_for(n, 256, 16), 256, 0, s>>>(field, n, cut);
  return sr_launch_status();
}
