// Weight gradients of the dense layers on the tensor cores (training half of the hot path:
// model/network.py:599-639 loss.backward(), :774-796 parameter VJPs of the implicit differentiation).
//
//   dW[n][k] = sum_rows delta[row][n] * x[row][k]          (rows = points x (value + tangent rows))
//
// Both operands already exist as tiled split-bf16 activations (tc_common.cuh): `x` = the layer's input tiles
// the forward sweep kept, `delta` = the cotangent tiles the reverse sweep wrote.  In that layout a core matrix
// is 8 rows x 8 features with the FEATURES contiguous, which is exactly the canonical MN-major core matrix of
// a wgmma operand whose GEMM-K dimension is the ROW index -- so the same bytes feed this GEMM as transposed
// (MN-major) A and B operands and no transposition pass is needed:
//      D[64 delta-features x 256 x-features] += A^T[64 x 16 rows] * B[16 rows x 256]
// per `wgmma.mma_async m64n256k16` and warpgroup, 3 MMAs per product (split-bf16 cross terms, as in tc_gemm.cu).
//
// One CTA owns one (128 x 256) tile of dW and a contiguous range of row half-tiles (split-K over points):
//   warp 0          TMA producer: a stage = 64 rows; per stage 32 + 64 bulk copies of 1 KB (one k8 group of one
//                   plane each) land the planes of 128 + 256 features separately, so that the feature stride is
//                   uniform (SBO = 1 KB, LBO = 128 B); the 32 lanes issue the copies in parallel
//   warpgroups 1-2  delta features [0, 64) / [64, 128) of the tile: MMAs into registers; every kFlush stages the
//                   accumulator is added to the CTA's fp32 partial tile in global memory with plain
//                   read-modify-write (each element is always handled by the same thread: deterministic).  Bounding
//                   the run length of an accumulator bounds the truncation bias of the tensor core's fp32 adder
//                   (tc_gemm.cu header): 16 stages = 1024 rows = 192 accumulations per element.
// A second kernel adds the split partials in a fixed order into dW (row-major [n][k], nn.Linear.weight's layout).
// The bias gradient (column sums of delta over VALUE rows) is a separate streaming kernel.
#include <cstdlib>

#include "tc_common.cuh"

namespace sr_tc {

constexpr int WG_ROWS = 64;                         // rows per stage (half a row tile)
constexpr int WG_STAGES = 2;
constexpr int WG_A_PLANE_BYTES = 16 * 1024;         // 128 features x 64 rows x 2 B
constexpr int WG_B_PLANE_BYTES = 32 * 1024;         // 256 features x 64 rows x 2 B
constexpr int WG_STAGE_BYTES = kPlanes * (WG_A_PLANE_BYTES + WG_B_PLANE_BYTES);   // 96 KB
constexpr size_t kSmemWgrad = (size_t)WG_STAGES * WG_STAGE_BYTES + 256;
constexpr int kFlush = 16;                          // stages per accumulator run
constexpr int kWgThreads = 3 * 128;
constexpr int kWgConsumerWarps = 8;
static_assert(kPlanes == 2, "the weight-gradient kernel is written for 2 planes / 3 terms");

struct WgradArgs {
  const __nv_bfloat16* D;   // delta tiles [MT][KCd][planes][128x32]
  const __nv_bfloat16* X;   // input tiles [MT][KCx][planes][128x32]
  int MT, KCd, KCx;
  int tiles_n;              // ceil(KCx / 8)
  int splits;
  float* part;              // [splits][KCd*32][KCx*32] fp32 partial sums
  int desc_swap;            // debugging aid: swap the LBO / SBO fields of the descriptors
};

// one stage (64 rows) of this warpgroup's 64 x 256 accumulator: 3 terms x 4 row steps of 16
template <bool FIRST>
__device__ __forceinline__ void wgrad_stage(float (&acc)[128], uint32_t abase, uint32_t bbase, uint32_t lbo,
                                            uint32_t sbo) {
  const int pa[3] = {0, 1, 0}, pb[3] = {1, 0, 0};   // smallest contributions first
#pragma unroll
  for (int q = 0; q < 3; ++q) {
#pragma unroll
    for (int j = 0; j < WG_ROWS / 16; ++j) {
      const uint64_t ad = make_desc(abase + pa[q] * WG_A_PLANE_BYTES + j * 256, lbo, sbo);
      const uint64_t bd = make_desc(bbase + pb[q] * WG_B_PLANE_BYTES + j * 256, lbo, sbo);
      if (FIRST && q == 0 && j == 0) wgmma_m64n256k16<1, 1, true>(acc, ad, bd);
      else wgmma_m64n256k16<1, 1, false>(acc, ad, bd);
    }
  }
}

__global__ void __launch_bounds__(kWgThreads, 1) tc_wgrad_kernel(const __grid_constant__ WgradArgs a) {
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)WG_STAGES * WG_STAGE_BYTES);
  uint64_t* full = bars;                  // [WG_STAGES]
  uint64_t* empty = bars + WG_STAGES;     // [WG_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    for (int i = 0; i < WG_STAGES; ++i) { sr_mbar_init(&full[i], 1); sr_mbar_init(&empty[i], kWgConsumerWarps); }
    sr_fence_barrier_init();
  }
  __syncthreads();

  const int tile = blockIdx.x / a.splits, split = blockIdx.x % a.splits;
  const int tm = tile / a.tiles_n, tn = tile % a.tiles_n;
  const int nb = min(8, a.KCx - tn * 8);              // 32-feature chunks of x in this tile; the MMA always runs
                                                      // N = 256: columns past 32 nb see stale shared memory and are
                                                      // never stored
  const int na = min(4, a.KCd - tm * 4);              // 32-feature chunks of delta in this tile (same for rows)
  const int halves = 2 * a.MT;
  const int per = (halves + a.splits - 1) / a.splits;
  const int h0 = split * per, h1 = min(halves, h0 + per);
  const int nstages = h1 > h0 ? h1 - h0 : 0;
  const int nruns = (nstages + kFlush - 1) / kFlush;

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer (32 lanes issue copies)
    int slot = 0;
    uint32_t phase = 0;
    for (int h = h0; h < h1; ++h) {
      const long long mt = h >> 1;
      const int half = h & 1;
      if (lane == 0) {
        sr_mbar_wait(&empty[slot], phase ^ 1u);
        sr_mbar_arrive_expect_tx(&full[slot], (uint32_t)(na * 8 + nb * 8) * 1024u);
      }
      __syncwarp();
      unsigned char* st = smem + (size_t)slot * WG_STAGE_BYTES;
      {  // delta: plane p, feature group g (8 features) of this tile's 128
        const int p = lane >> 4, g = lane & 15;
        if ((g >> 2) < na) {
          const __nv_bfloat16* src = a.D + a_tile_off(mt, tm * 4 + (g >> 2), a.KCd, p) + (size_t)(g & 3) * (BM * 8) +
                                     (size_t)half * (WG_ROWS * 8);
          sr_bulk_g2s(st + p * WG_A_PLANE_BYTES + g * 1024, src, 1024u, &full[slot]);
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = lane + 32 * i, p = c >> 5, g = c & 31;
        if ((g >> 2) < nb) {
          const __nv_bfloat16* src = a.X + a_tile_off(mt, tn * 8 + (g >> 2), a.KCx, p) +
                                     (size_t)(g & 3) * (BM * 8) + (size_t)half * (WG_ROWS * 8);
          sr_bulk_g2s(st + kPlanes * WG_A_PLANE_BYTES + p * WG_B_PLANE_BYTES + g * 1024, src, 1024u, &full[slot]);
        }
      }
      if (++slot == WG_STAGES) { slot = 0; phase ^= 1u; }
    }
  } else if (wg > 0) {
    // ------------------------------------------------------------------ MMA + drain (warpgroups 1, 2)
    const int cw = wg - 1, wq = warp & 3;
    const uint32_t lbo = a.desc_swap ? 1024u : 128u, sbo = a.desc_swap ? 128u : 1024u;
    // fragment rows (delta features) 16 wq + lane / 4 (+ 8) of this warpgroup's 64, columns 8 i + 2 (lane % 4) (+ 1)
    const int row0 = tm * 128 + cw * 64 + 16 * wq + (lane >> 2);
    const size_t ld = (size_t)a.KCx * 32;
    float* dst0 = a.part + ((size_t)split * ((size_t)a.KCd * 32) + row0) * ld + (size_t)tn * 256 + 2 * (lane & 3);
    const bool ok0 = row0 < a.KCd * 32, ok1 = row0 + 8 < a.KCd * 32;
    const int ncols8 = 4 * nb;                        // stored 8-column blocks
    float acc[128];
    int slot = 0;
    uint32_t phase = 0;
    int s = 0;
    // operands of stage `slot`: this warpgroup's 64 delta features (8 groups of 8) and the 256 x features
    auto abase = [&](int sl) { return sr_smem_u32(smem + (size_t)sl * WG_STAGE_BYTES) + cw * 8 * 1024; };
    auto bbase = [&](int sl) { return sr_smem_u32(smem + (size_t)sl * WG_STAGE_BYTES) + kPlanes * WG_A_PLANE_BYTES; };
    for (int run = 0; run < nruns; ++run) {
      const int s_end = min(nstages, s + kFlush);
      // the first stage of a run overwrites the accumulator (peeled: no data-dependent branch around the MMAs)
      sr_mbar_wait(&full[slot], phase);
      wgmma_fence();
      wgrad_stage<true>(acc, abase(slot), bbase(slot), lbo, sbo);
      wgmma_commit();
      int prev = slot;
      if (++slot == WG_STAGES) { slot = 0; phase ^= 1u; }
      for (++s; s < s_end; ++s) {
        sr_mbar_wait(&full[slot], phase);
        wgmma_fence();
        wgrad_stage<false>(acc, abase(slot), bbase(slot), lbo, sbo);
        wgmma_commit();
        wgmma_wait<1>();   // the previous stage's MMAs are complete: release it
        if (lane == 0) sr_mbar_arrive(&empty[prev]);
        prev = slot;
        if (++slot == WG_STAGES) { slot = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      if (lane == 0) sr_mbar_arrive(&empty[prev]);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        if (i >= ncols8) break;
        float2 o0 = make_float2(acc[4 * i], acc[4 * i + 1]), o1 = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
        float2* d0 = reinterpret_cast<float2*>(dst0 + 8 * i);
        float2* d1 = reinterpret_cast<float2*>(dst0 + 8 * ld + 8 * i);
        if (run > 0) {
          if (ok0) { const float2 t = *d0; o0.x += t.x; o0.y += t.y; }
          if (ok1) { const float2 t = *d1; o1.x += t.x; o1.y += t.y; }
        }
        if (ok0) *d0 = o0;
        if (ok1) *d1 = o1;
      }
    }
    if (nruns == 0) {   // a split without rows still owns its partial tile
      for (int i = 0; i < ncols8; ++i) {
        if (ok0) *reinterpret_cast<float2*>(dst0 + 8 * i) = make_float2(0.f, 0.f);
        if (ok1) *reinterpret_cast<float2*>(dst0 + 8 * ld + 8 * i) = make_float2(0.f, 0.f);
      }
    }
  }
}

// dW[n][k] (ld) = sum_s part[s][n][k] for n < N, k < K, fixed order
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ part, int splits, int rows_pad, int cols_pad, float* __restrict__ dW,
                    int N, int K, int ld) {
  const long long total = (long long)N * K;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(idx / K), k = (int)(idx % K);
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += part[((size_t)s * rows_pad + n) * cols_pad + k];
    dW[(size_t)n * ld + k] = acc;
  }
}

// column sums of the tiled activations over rows with row % ch == 0: out[part][k]; one block = (chunk kc,
// slice of row tiles); fp32 adds in a fixed order, partial sums reduced by the caller
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ T, int MT, int KC, int ch, int slices, float* __restrict__ out) {
  const int kc = blockIdx.x % KC, slice = blockIdx.x / KC;
  const int per = (MT + slices - 1) / slices;
  const int m0 = slice * per, m1 = min(MT, m0 + per);
  const int k = threadIdx.x & 31, rq = threadIdx.x >> 5;      // 32 features x 8 row phases
  float acc = 0.f;
  for (int mt = m0; mt < m1; ++mt) {
    const __nv_bfloat16* t0 = T + a_tile_off(mt, kc, KC, 0);
    for (int r = rq * ch; r < BM; r += 8 * ch) {
      const int off = (k >> 3) * (BM * 8) + (r >> 3) * 64 + (r & 7) * 8 + (k & 7);
      acc += __bfloat162float(t0[off]) + __bfloat162float(t0[off + A_PLANE]);
    }
  }
  __shared__ float red[8][32];
  red[rq][k] = acc;
  __syncthreads();
  if (rq == 0) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][k];
    out[(size_t)slice * (KC * 32) + kc * 32 + k] = s;
  }
}

// tiled split-bf16 rows -> fp32 row-major [M][K] (ld): the inverse of pack_rows (tests, debugging)
__global__ void unpack_rows_kernel(const __nv_bfloat16* __restrict__ T, long long M, int K, int KC,
                                   float* __restrict__ out, int ld) {
  const long long total = M * (long long)K;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / K;
    const int k = (int)(idx % K);
    const long long mt = row / BM;
    const int r = (int)(row % BM);
    const __nv_bfloat16* t0 = T + a_tile_off(mt, k >> 5, KC, 0);
    const int kk = k & 31;
    const int off = (kk >> 3) * (BM * 8) + (r >> 3) * 64 + (r & 7) * 8 + (kk & 7);
    out[(size_t)row * ld + k] = __bfloat162float(t0[off]) + __bfloat162float(t0[off + A_PLANE]);
  }
}

}  // namespace sr_tc

static int g_wgrad_desc_swap = 0;

extern "C" {

// Debug knob (tests): 1 swaps the LBO / SBO fields of the MN-major operand descriptors.
void sr_tc_debug_wgrad_desc_swap(int v) { g_wgrad_desc_swap = v; }

int64_t sr_tc_wgrad_partial_bytes(int64_t M, int Kd, int Kx, int* splits_out) {
  using namespace sr_tc;
  const int MT = (int)((M + BM - 1) / BM), KCd = (Kd + 31) / 32, KCx = (Kx + 31) / 32;
  const int tiles = ((KCd + 3) / 4) * ((KCx + 7) / 8);
  int splits = SR_NUM_SMS / (tiles > 0 ? tiles : 1);
  if (splits < 1) splits = 1;
  if (splits > 2 * MT) splits = 2 * MT;
  if (splits_out) *splits_out = splits;
  return (int64_t)splits * KCd * 32 * KCx * 32 * 4;
}

int sr_tc_wgrad(const void* D, int Kd, const void* X, int Kx, int64_t M, float* part, float* dW, int N, int K,
                int ld, cudaStream_t s) {
  using namespace sr_tc;
  if (!D || !X || !part || !dW || M <= 0 || Kd <= 0 || Kx <= 0 || N <= 0 || K <= 0 || ld < K) return SR_EINVAL;
  WgradArgs a;
  a.D = (const __nv_bfloat16*)D; a.X = (const __nv_bfloat16*)X;
  a.MT = (int)((M + BM - 1) / BM); a.KCd = (Kd + 31) / 32; a.KCx = (Kx + 31) / 32;
  if (N > a.KCd * 32 || K > a.KCx * 32) return SR_EINVAL;
  a.tiles_n = (a.KCx + 7) / 8;
  int splits = 1;
  sr_tc_wgrad_partial_bytes(M, Kd, Kx, &splits);
  a.splits = splits; a.part = part;
  a.desc_swap = g_wgrad_desc_swap;
  static bool attr_set_dev[64] = {};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  if (!attr_set_dev[cur_dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(tc_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemWgrad);
    if (e != cudaSuccess) return (int)e;
    attr_set_dev[cur_dev & 63] = true;
  }
  const int tiles = ((a.KCd + 3) / 4) * a.tiles_n;
  tc_wgrad_kernel<<<tiles * splits, kWgThreads, kSmemWgrad, s>>>(a);
  int rc = sr_launch_status();
  if (rc) return rc;
  const long long total = (long long)N * K;
  wgrad_reduce_kernel<<<sr_grid_for(total, 256, 8), 256, 0, s>>>(part, splits, a.KCd * 32, a.KCx * 32, dW, N, K, ld);
  return sr_launch_status();
}

int sr_tc_colsum(const void* T, int64_t M, int K, int ch, float* partial, int slices, cudaStream_t s) {
  using namespace sr_tc;
  if (!T || !partial || M <= 0 || K <= 0 || (ch != 1 && ch != 4) || slices <= 0) return SR_EINVAL;
  const int MT = (int)((M + BM - 1) / BM), KC = (K + 31) / 32;
  colsum_kernel<<<KC * slices, 256, 0, s>>>((const __nv_bfloat16*)T, MT, KC, ch, slices, partial);
  return sr_launch_status();
}

int sr_tc_unpack_rows(const void* T, int64_t M, int K, int Kpad, float* out, int ld, cudaStream_t s) {
  using namespace sr_tc;
  if (!T || !out || M <= 0 || K <= 0 || Kpad < K || ld < K) return SR_EINVAL;
  unpack_rows_kernel<<<sr_grid_for(M * (long long)K, 256, 8), 256, 0, s>>>((const __nv_bfloat16*)T, M, K,
                                                                          (Kpad + 31) / 32, out, ld);
  return sr_launch_status();
}
}

// ---- whole-sweep entry points ---------------------------------------------------------------------
// One C call per forward / backward sweep of an MLP: the per-layer launches above are issued from here, so the host
// cost of a training evaluation is one FFI crossing instead of ~5 per layer (the 8192-ray training step was bound by
// Python launch overhead: ~700 own launches per step).
namespace sr_tc {

__global__ void colsum_reduce_kernel(const float* __restrict__ partial, int slices, int ld, float* __restrict__ out, int n) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  float acc = 0.f;
  for (int s = 0; s < slices; ++s) acc += partial[(size_t)s * ld + k];
  out[k] = acc;
}

__global__ void add_cols_kernel(float* __restrict__ dst, int ld_dst, const float* __restrict__ src, int ld_src, long long M,
                                int n) {
  const long long total = M * n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / n;
    const int c = (int)(idx % n);
    dst[r * ld_dst + c] += src[r * ld_src + c];
  }
}

__global__ void zero_cols_kernel(float* __restrict__ dst, int ld, long long M, int c0, int c1) {
  const int w = c1 - c0;
  const long long total = M * w;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x)
    dst[(idx / w) * ld + c0 + (int)(idx % w)] = 0.f;
}

}  // namespace sr_tc

extern "C" {

int sr_tc_linear(const void* A, const void* W, const float* bias, int64_t M, int N, int K, int n_valid, int act, int ch,
                 void* A_next, int K_next, float scale, const float* skip_src, int skip_n, int skip_ld, float* out,
                 int out_ld, int out_col0, int out_n, float* dstash, const void* mul_tiles, int mul_K, int mul_act,
                 float mul_scale, const int32_t* m_dev, cudaStream_t s);
int sr_tc_pack_rows(const float* src, int64_t M, int K, int ld, void* dst, const int32_t* m_dev, cudaStream_t s);

static inline int pad_to(int x, int m) { return (x + m - 1) / m * m; }

int sr_tc_mlp_forward(const sr_tc_layer* layers, int L, const float* x0, int64_t M, int ld, int d_in, int ch, void* A_in,
                      void* const* acts, float* const* stashes, float* out, const int32_t* m_dev, int n_out,
                      cudaStream_t s) {
  if (!layers || L <= 0 || L > 16 || !x0 || M <= 0 || ld <= 0 || (ld % 32) != 0 || !A_in || !out || (L > 1 && !acts) ||
      n_out < 0 || n_out > layers[L - 1].n)
    return SR_EINVAL;
  int rc = sr_tc_pack_rows(x0, M, ld, ld, A_in, m_dev, s);
  if (rc) return rc;
  const void* cur = A_in;
  int K = ld;
  for (int i = 0; i < L; ++i) {
    const sr_tc_layer& ly = layers[i];
    const bool last = i == L - 1;
    const bool skip_next = !last && layers[i + 1].skip;
    const int Kn = last ? 0 : pad_to(layers[i + 1].k, 32);
    const int nv = last && n_out > 0 ? n_out : ly.n;
    rc = sr_tc_linear(cur, ly.W, ly.bias, M, ly.n, K, nv, ly.act, ch, last ? nullptr : acts[i], Kn,
                      skip_next ? 0.70710678118654752f : 1.0f, skip_next ? x0 : nullptr, skip_next ? d_in : 0, ld,
                      last ? out : nullptr, last ? nv : 0, 0, nv, (!last && stashes) ? stashes[i] : nullptr, nullptr, 0,
                      0, 1.0f, m_dev, s);
    if (rc) return rc;
    if (!last) { cur = acts[i]; K = Kn; }
  }
  return SR_OK;
}

int sr_tc_mlp_backward(const sr_tc_layer* layers, int L, int64_t M, int ld, int d_in, int ch, const float* gout,
                       const void* A_in, void* const* acts, float* const* stashes, void* D0, void* D1, float* part,
                       float* colsum_ws, int colsum_slices, float* const* dW, float* const* db, float* x0_grad,
                       float* g_skip, int g_skip_ld, cudaStream_t s) {
  using namespace sr_tc;
  if (!layers || L <= 0 || L > 16 || M <= 0 || !gout || !A_in || !D0 || !D1 || !part || !colsum_ws || !dW || !db)
    return SR_EINVAL;
  const int n_last = layers[L - 1].n;
  int Kd = pad_to(n_last, 32);
  void* D = D0;
  void* Dn = D1;
  int rc = sr_tc_pack_rows(gout, M, n_last, n_last, D, nullptr, s);
  if (rc) return rc;
  bool had_skip = false;
  for (int l = L - 1; l >= 0; --l) {
    const sr_tc_layer& ly = layers[l];
    const void* X = l > 0 ? acts[l - 1] : A_in;
    const int Kx = l > 0 ? pad_to(ly.k, 32) : ld;
    if (dW[l]) {
      rc = sr_tc_wgrad(D, Kd, X, Kx, M, part, dW[l], ly.n, ly.k, ly.k, s);
      if (rc) return rc;
    }
    if (db[l]) {
      rc = sr_tc_colsum(D, M, Kd, ch, colsum_ws, colsum_slices, s);
      if (rc) return rc;
      colsum_reduce_kernel<<<(ly.n + 127) / 128, 128, 0, s>>>(colsum_ws, colsum_slices, Kd, db[l], ly.n);
    }
    if (l == 0 && !x0_grad) break;
    const float scale = ly.skip ? 0.70710678118654752f : 1.0f;
    if (l > 0) {
      const int n_prev = layers[l - 1].n;
      const int Kd_prev = pad_to(n_prev, 32);
      if (ly.skip && !g_skip) return SR_EINVAL;
      rc = sr_tc_linear(D, ly.Wb, ly.zero_bias, M, ly.k, Kd, n_prev, SR_ACT_NONE, ch, Dn, Kd_prev, scale, nullptr, 0, 0,
                        ly.skip ? g_skip : nullptr, ly.skip ? g_skip_ld : 0, n_prev, ly.skip ? d_in : 0,
                        stashes ? stashes[l - 1] : nullptr, acts[l - 1], pad_to(ly.k, 32), layers[l - 1].act, scale, nullptr,
                        s);
      if (rc) return rc;
      had_skip |= ly.skip != 0;
      void* t = D; D = Dn; Dn = t;
      Kd = Kd_prev;
    } else {
      rc = sr_tc_linear(D, ly.Wb, ly.zero_bias, M, ly.k, Kd, ly.k, SR_ACT_NONE, 1, nullptr, 0, scale, nullptr, 0, 0, x0_grad,
                        ld, 0, ly.k, nullptr, nullptr, 0, 0, 1.0f, nullptr, s);
      if (rc) return rc;
      if (ly.k < ld) zero_cols_kernel<<<sr_grid_for(M * (ld - ly.k), 256, 4), 256, 0, s>>>(x0_grad, ld, M, ly.k, ld);
      if (had_skip)
        add_cols_kernel<<<sr_grid_for(M * d_in, 256, 4), 256, 0, s>>>(x0_grad, ld, g_skip, g_skip_ld, M, d_in);
    }
  }
  return sr_launch_status();
}
}
