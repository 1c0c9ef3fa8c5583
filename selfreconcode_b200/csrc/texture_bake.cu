// Texture atlas of the reconstruction (the reference's texture_mesh_extract.py:57-144, VideoAvatar's Isomapper step),
// per texel on the device.  The atlas texels a UV face covers are listed once (the UV raster, csrc/raster.cu on the
// atlas), so both kernels run over that compacted list: T covered texels, S slots each.
//
// Slots are slot-major ([S][T]) so that thread t's access to slot s of texel t is coalesced across the warp:
//   slot_rgb   [S][3][T] float   colour (planar per channel)
//   slot_alpha [S][T]    float   view weight, c0 = cos(max_angle) when empty
//   slot_view  [S][T]    int32   frame id, -1 when empty
// plus a per-texel (min alpha, first slot holding it) pair, so that a frame reads 24 B per covered texel (face id,
// barycentrics, the pair) and only a texel whose slot is replaced touches its slots (12 + 4 + 4 B written, S alphas
// rescanned for the new minimum).
//
// sr_texture_accumulate (one frame, one thread per texel; texture_mesh_extract.py:101-123):
//   face k usable, barycentrics b:  alpha = sum b_i a[F[k][i]];  p = sum b_i s[F[k][i]]  (pixel centres at integers)
//   if alpha > min alpha: slot <- (bilinear(image, p) / 255 with clamp-to-edge, alpha, frame id), new min rescanned.
//   Texels of unusable faces have alpha 0 and never enter (the slots start at c0 > 0).
// sr_texture_finish (one thread per texel; :131-144):  count = #slots with alpha > c0, mask_final = count >= min_views,
//   view_id = frame of the first slot with the largest alpha, per-channel median of the filled slots (np.nanmedian: the
//   mean of the two middle values for an even count), sorted by insertion in a shared-memory column of the thread (up
//   to SR_TEXTURE_MAX_SLOTS values, thread-major so the column accesses are free of bank conflicts; nothing spills).
// Every texel is owned by one thread in both kernels: no atomics, bit-identical reruns.
#include "common.cuh"

namespace {

constexpr int kFinishThreads = 128;

__device__ __forceinline__ float texel_at(const unsigned char* __restrict__ img, int W, int r, int c, int ch) {
  return (float)img[((long long)r * W + c) * 3 + ch];
}

__global__ void __launch_bounds__(256)
texture_accumulate_kernel(long long T, int S, const int* __restrict__ texel_face, const float* __restrict__ texel_bary,
                          const float* __restrict__ vs, const long long* __restrict__ faces, long long V, long long F,
                          const float* __restrict__ weight, const unsigned char* __restrict__ usable,
                          const unsigned char* __restrict__ img, int H, int W, int frame_id,
                          float* __restrict__ slot_rgb, float* __restrict__ slot_alpha, int* __restrict__ slot_view,
                          float* __restrict__ min_alpha, int* __restrict__ min_slot) {
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (long long)gridDim.x * blockDim.x) {
    const int k = texel_face[t];
    if (k < 0 || k >= F || !usable[k]) continue;
    const long long i0 = faces[k * 3], i1 = faces[k * 3 + 1], i2 = faces[k * 3 + 2];
    if (i0 < 0 || i0 >= V || i1 < 0 || i1 >= V || i2 < 0 || i2 >= V) continue;
    const float b0 = texel_bary[t * 3], b1 = texel_bary[t * 3 + 1], b2 = texel_bary[t * 3 + 2];
    const float alpha = b0 * weight[i0] + b1 * weight[i1] + b2 * weight[i2];
    if (!(alpha > min_alpha[t])) continue;
    const int s = min_slot[t];
    // bilinear sample at p (clamped to [-1, W] x [-1, H] first: clamp-to-edge gives the same value, and the float ->
    // int conversion stays defined for any p)
    float px = b0 * vs[i0 * 3] + b1 * vs[i1 * 3] + b2 * vs[i2 * 3];
    float py = b0 * vs[i0 * 3 + 1] + b1 * vs[i1 * 3 + 1] + b2 * vs[i2 * 3 + 1];
    px = fminf(fmaxf(px, -1.f), (float)W);
    py = fminf(fmaxf(py, -1.f), (float)H);
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float fx = px - fx0, fy = py - fy0;
    const int x0 = min(max((int)fx0, 0), W - 1), x1 = min(max((int)fx0 + 1, 0), W - 1);
    const int y0 = min(max((int)fy0, 0), H - 1), y1 = min(max((int)fy0 + 1, 0), H - 1);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float top = (1.f - fx) * texel_at(img, W, y0, x0, ch) + fx * texel_at(img, W, y0, x1, ch);
      const float bot = (1.f - fx) * texel_at(img, W, y1, x0, ch) + fx * texel_at(img, W, y1, x1, ch);
      slot_rgb[((long long)s * 3 + ch) * T + t] = ((1.f - fy) * top + fy * bot) / 255.f;
    }
    slot_alpha[(long long)s * T + t] = alpha;
    slot_view[(long long)s * T + t] = frame_id;
    // new (min, first slot holding it)
    float m = alpha;
    int ms = s;
    for (int j = 0; j < S; ++j) {
      const float v = j == s ? alpha : slot_alpha[(long long)j * T + t];
      if (v < m || (v == m && j < ms)) {
        m = v;
        ms = j;
      }
    }
    min_alpha[t] = m;
    min_slot[t] = ms;
  }
}

__global__ void __launch_bounds__(kFinishThreads)
texture_finish_kernel(long long T, int S, const long long* __restrict__ texel_index, const float* __restrict__ slot_rgb,
                      const float* __restrict__ slot_alpha, const int* __restrict__ slot_view, float c0,
                      int min_views, float* __restrict__ tex_median, unsigned char* __restrict__ mask_final,
                      int* __restrict__ view_id, int* __restrict__ count) {
  __shared__ float col[SR_TEXTURE_MAX_SLOTS * kFinishThreads];
  float* my = col + threadIdx.x;       // element j at my[j * kFinishThreads]
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (long long)gridDim.x * blockDim.x) {
    unsigned long long filled = 0ULL;
    int n = 0, best_s = 0;
    float best = slot_alpha[t];
    for (int s = 0; s < S; ++s) {
      const float a = slot_alpha[(long long)s * T + t];
      if (a > c0) {
        filled |= 1ULL << s;
        ++n;
      }
      if (a > best) {
        best = a;
        best_s = s;
      }
    }
    const bool ok = n >= min_views;
    const long long o = texel_index[t];
    count[o] = n;
    mask_final[o] = ok ? 1 : 0;
    view_id[o] = ok ? slot_view[(long long)best_s * T + t] : -1;
    for (int ch = 0; ch < 3; ++ch) {
      float med = 0.f;
      if (ok) {
        int m = 0;
        for (int s = 0; s < S; ++s) {
          if (!((filled >> s) & 1ULL)) continue;
          const float v = slot_rgb[((long long)s * 3 + ch) * T + t];
          int j = m;
          while (j > 0 && my[(j - 1) * kFinishThreads] > v) {
            my[j * kFinishThreads] = my[(j - 1) * kFinishThreads];
            --j;
          }
          my[j * kFinishThreads] = v;
          ++m;
        }
        const int h = n >> 1;
        med = (n & 1) ? my[h * kFinishThreads] : 0.5f * (my[(h - 1) * kFinishThreads] + my[h * kFinishThreads]);
      }
      tex_median[o * 3 + ch] = med;
    }
  }
}

}  // namespace

extern "C" int sr_texture_accumulate(int64_t T, int S, const int32_t* texel_face, const float* texel_bary,
                                     const float* verts_screen, const int64_t* faces, int64_t V, int64_t F,
                                     const float* vert_weight, const uint8_t* face_usable, const uint8_t* image, int H,
                                     int W, int frame_id, float* slot_rgb, float* slot_alpha, int32_t* slot_view,
                                     float* min_alpha, int32_t* min_slot, cudaStream_t s) {
  if (!texel_face || !texel_bary || !verts_screen || !faces || !vert_weight || !face_usable || !image || !slot_rgb ||
      !slot_alpha || !slot_view || !min_alpha || !min_slot || T <= 0 || S <= 0 || S > SR_TEXTURE_MAX_SLOTS || V <= 0 ||
      F <= 0 || F > 0x7fffffffLL || H <= 0 || W <= 0 || frame_id < 0)
    return SR_EINVAL;
  texture_accumulate_kernel<<<sr_grid_for(T, 256, 8), 256, 0, s>>>(
      T, S, texel_face, texel_bary, verts_screen, (const long long*)faces, V, F, vert_weight, face_usable, image, H, W,
      frame_id, slot_rgb, slot_alpha, slot_view, min_alpha, min_slot);
  return sr_launch_status();
}

extern "C" int sr_texture_finish(int64_t T, int S, const int64_t* texel_index, const float* slot_rgb,
                                 const float* slot_alpha, const int32_t* slot_view, float c0, int min_views,
                                 float* tex_median, uint8_t* mask_final, int32_t* view_id, int32_t* count,
                                 cudaStream_t s) {
  if (!texel_index || !slot_rgb || !slot_alpha || !slot_view || !tex_median || !mask_final || !view_id || !count ||
      T <= 0 || S <= 0 || S > SR_TEXTURE_MAX_SLOTS || min_views < 1 || min_views > S || !(c0 > 0.f && c0 < 1.f))
    return SR_EINVAL;
  texture_finish_kernel<<<sr_grid_for(T, kFinishThreads, 8), kFinishThreads, 0, s>>>(
      T, S, (const long long*)texel_index, slot_rgb, slot_alpha, slot_view, c0, min_views, tex_median, mask_final,
      view_id, count);
  return sr_launch_status();
}
