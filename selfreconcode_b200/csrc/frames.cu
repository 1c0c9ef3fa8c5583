// Decode of a training batch from the device-resident frame store (dataset/dataset.py:89-102 of the reference:
// SceneDataset.__getitem__, whose cv2 decode runs once per sequence on the host instead of once per step).
//
// One thread turns 4 consecutive pixels of a frame into 12 + 4 + 12 floats: it reads 12 B of image, 12 B of normal
// and one mask word and writes 112 B, as 16 B stores when a frame holds a multiple of 4 pixels (then every frame's
// byte planes start 4 B aligned and its fp32 planes 16 B aligned).  The pass is an HBM stream: 6.1 B read and 28 B
// written per pixel.  Every fp32 operation is its own correctly rounded intrinsic, so nvcc cannot contract them and
// the values are bit-identical to numpy's float32 expressions.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float img_value(uint32_t x) {   // (x / 255. - 0.5) * 2 in float32
  return __fmul_rn(__fsub_rn(__fdiv_rn((float)x, 255.f), 0.5f), 2.f);
}
__device__ __forceinline__ float normal_value(uint32_t x) {  // 2. * x / 255. - 1. in float32
  return __fsub_rn(__fdiv_rn(__fmul_rn(2.f, (float)x), 255.f), 1.f);
}

template <bool kVec>
__global__ void __launch_bounds__(kThreads)
frames_decode_kernel(const uint8_t* __restrict__ img_store, const uint32_t* __restrict__ mask_store,
                     const uint8_t* __restrict__ normal_store, int F, int H, int W,
                     const int64_t* __restrict__ frame_ids, int64_t N, float* __restrict__ img,
                     float* __restrict__ mask, float* __restrict__ normal) {
  const int64_t HW = (int64_t)H * W;
  const int64_t groups = (HW + 3) >> 2;
  const int Wd = (W + 31) >> 5;
  for (int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x; t < N * groups;
       t += (int64_t)gridDim.x * kThreads) {
    const int64_t n = t / groups;
    const int64_t q = (t - n * groups) << 2;  // first pixel of the group within its frame
    const int64_t f = frame_ids[n];
    if (f < 0 || f >= F) continue;
    const int cnt = kVec ? 4 : (int)min((int64_t)4, HW - q);
    const int64_t src = f * HW + q, dst = n * HW + q;
    if (img) {
      uint8_t b[12];
      if (kVec) {
        const uint32_t* s = reinterpret_cast<const uint32_t*>(img_store + src * 3);
#pragma unroll
        for (int k = 0; k < 3; ++k) *reinterpret_cast<uint32_t*>(b + 4 * k) = __ldg(s + k);
      } else {
#pragma unroll
        for (int k = 0; k < 12; ++k) b[k] = k < 3 * cnt ? img_store[src * 3 + k] : 0;
      }
      float o[12];
#pragma unroll
      for (int k = 0; k < 12; ++k) o[k] = img_value(b[k]);
      if (kVec) {
        float4* d = reinterpret_cast<float4*>(img + dst * 3);
#pragma unroll
        for (int k = 0; k < 3; ++k) d[k] = make_float4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
      } else {
#pragma unroll
        for (int k = 0; k < 12; ++k)
          if (k < 3 * cnt) img[dst * 3 + k] = o[k];
      }
    }
    if (normal) {
      uint8_t b[12];
      if (kVec) {
        const uint32_t* s = reinterpret_cast<const uint32_t*>(normal_store + src * 3);
#pragma unroll
        for (int k = 0; k < 3; ++k) *reinterpret_cast<uint32_t*>(b + 4 * k) = __ldg(s + k);
      } else {
#pragma unroll
        for (int k = 0; k < 12; ++k) b[k] = k < 3 * cnt ? normal_store[src * 3 + k] : 0;
      }
      float o[12];
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int c = 0; c < 3; ++c) o[3 * p + c] = normal_value(b[3 * p + 2 - c]);  // BGR -> RGB
      if (kVec) {
        float4* d = reinterpret_cast<float4*>(normal + dst * 3);
#pragma unroll
        for (int k = 0; k < 3; ++k) d[k] = make_float4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
      } else {
#pragma unroll
        for (int k = 0; k < 12; ++k)
          if (k < 3 * cnt) normal[dst * 3 + k] = o[k];
      }
    }
    if (mask) {
      float o[4];
      int64_t r = q / W;
      int c = (int)(q - r * W);
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        o[p] = 0.f;
        if (p < cnt) {
          const uint32_t w = __ldg(mask_store + (f * H + r) * Wd + (c >> 5));
          o[p] = ((w >> (c & 31)) & 1u) ? 1.f : 0.f;
        }
        if (++c == W) {  // the group runs into the next row
          c = 0;
          ++r;
        }
      }
      if (kVec) {
        *reinterpret_cast<float4*>(mask + dst) = make_float4(o[0], o[1], o[2], o[3]);
      } else {
#pragma unroll
        for (int p = 0; p < 4; ++p)
          if (p < cnt) mask[dst + p] = o[p];
      }
    }
  }
}

}  // namespace

extern "C" int sr_frames_decode(const uint8_t* img_store, const uint32_t* mask_store, const uint8_t* normal_store,
                                int F, int H, int W, const int64_t* frame_ids, int64_t N, float* img, float* mask,
                                float* normal, cudaStream_t s) {
  if (F <= 0 || H <= 0 || W <= 0 || N < 0) return SR_EINVAL;
  if ((img && !img_store) || (mask && !mask_store) || (normal && !normal_store)) return SR_EINVAL;
  if (N == 0 || (!img && !mask && !normal)) return SR_OK;
  if (!frame_ids) return SR_EINVAL;
  const int64_t HW = (int64_t)H * W;
  const int64_t work = N * ((HW + 3) >> 2);
  const int grid = sr_grid_for(work, kThreads, 16);
  if (HW % 4 == 0)
    frames_decode_kernel<true><<<grid, kThreads, 0, s>>>(img_store, mask_store, normal_store, F, H, W, frame_ids, N,
                                                         img, mask, normal);
  else
    frames_decode_kernel<false><<<grid, kThreads, 0, s>>>(img_store, mask_store, normal_store, F, H, W, frame_ids,
                                                          N, img, mask, normal);
  return sr_launch_status();
}
