// Tensor-core engine for the dense layers: split-BF16 GEMM on Hopper wgmma with fp32 accumulation in
// registers (SURVEY.md section 7 "hard parts": the ray finder tests |f| < 5e-5; a single BF16 or TF32 pass
// does not hold that).  Every fp32 operand is split into bf16 planes x = b1 + b2 (+ b3) and the product is
// assembled from the leading cross terms:
//     2 planes / 3 MMAs (default):  x*w ~= b1w1 + b1w2 + b2w1         (dropped: <= 2^-16 relative)
//     3 planes / 6 MMAs (-DSR_TC_PLANES=3): + b2w2 + b1w3 + b3w1      (dropped: <= 2^-24 relative)
// The tensor core adds each MMA into the fp32 accumulator with truncation, so the error of a K=512 layer is
// dominated by the NUMBER of accumulations (K/16 per term) rather than by the dropped terms (tools/tc_terms.py
// compares the two builds).
//
// One launch runs one layer  C[M x N] = act(A[M x K] * W^T + b)  over all row tiles:
//   * operands live in global memory already in the canonical (no-swizzle, K-major) shared memory layout
//     of the wgmma descriptors -- 128-byte core matrices (8 rows x 8 bf16), tiles of 128 (or 256 / 64) rows
//     x 32 k, the split planes of a tile contiguous -- so ONE TMA bulk copy (cp.async.bulk + mbarrier)
//     per operand per stage lands a ready-to-use tile and no tensor map is needed.  The previous layer's
//     epilogue writes its output directly in that layout (activations stay L2-resident between layers
//     for the batch sizes used here);
//   * warp-specialised, persistent CTAs: warpgroup 0 = TMA producer, warpgroups 1-2 = wgmma on 64 rows
//     each, then the epilogue of those rows (bias, activation, forward-mode tangent scaling or
//     reverse-mode act' multiply, re-split to bf16 planes, tiled store); the epilogue is specialised at
//     compile time per (activation, rows-per-point, mode);
//   * 3-stage shared-memory ring of 48 KB stages (6 stages of 24 KB on the narrow column tile): the bulk copies of the next tile run under the epilogue, the
//     MMAs do not (both consumer warpgroups are in the epilogue of the same tile; DESIGN.md section 8).  A reverse
//     launch also streams the previous layer's activation tiles (act' is recomputed from them) through the ring,
//     as epilogue stages after each n-tile's k chunks, so the epilogue reads them from shared memory.
// The FFMA engine (mlp_kernels.cu) stays the accuracy reference; tests compare both.
#include <cstdlib>

#include "tc_common.cuh"

namespace sr_tc {

struct LayerArgs {
  const __nv_bfloat16* A;   // tiled activations  [MT][KC][3][128x32]
  const __nv_bfloat16* W;   // tiled weights      [NT][KC][planes][bn x 32], bn = tile_n(n_gemm)
  const float* bias;        // [pad256(n_gemm)]
  long long M;              // valid rows
  int MT, NT, KC;           // row tiles, col tiles (of bn columns), k chunks (K = 32*KC)
  int n_gemm;               // columns the GEMM produces (<= NT*bn); the MMAs always run N = bn over zero-padded
                            // weight rows, the epilogue skips the chunks past n_gemm
  int n;                    // valid output columns
  int ch;                   // rows per point: 1 (value only) or 4 (value + 3 tangents)
  // outputs (either may be null)
  __nv_bfloat16* A_next;    // tiled, KCn chunks: activations for the next layer
  int KCn;
  float scale;              // 1, or 1/sqrt(2) when the next layer is the skip layer
  const float* skip_src;    // fp32 [M][skip_ld] embedded input appended after column n (or null)
  int skip_n, skip_ld;
  float* out;               // fp32 row-major [M][out_ld] (last layer), columns [0, n)
  int out_ld;
  float* dstash;            // fp32 row-major act'(z) of value rows or null: written by a forward launch ([M][NT*256]),
                            // read by a reverse launch ([M][pad256(n)], the previous layer's forward stash)
  // reverse sweep (MUL kernels): out = acc * act'(z_prev), act' recomputed from the previous layer's
  // stored output a (the tiles the forward pass wrote for this layer's input, scaled by 1/mul_inv_scale):
  // softplus100: 1 - exp(-100 a), relu: a > 0
  const __nv_bfloat16* mul_tiles;
  int mul_KC;
  float mul_inv_scale;
  int out_col0;             // `out` receives columns [out_col0, out_col0 + out_n) of the result
  int out_n;
  const int* m_dev;         // optional device-side row count (active rays); M is the upper bound
};

template <int ACT>
__device__ __forceinline__ float act_fn(float z, float& d) {
  if constexpr (ACT == SR_ACT_SOFTPLUS100) {
    const float bz = z * 100.0f;
    const float e = __expf(fminf(bz, 20.0f));
    const float sp = __logf(1.0f + e) * 0.01f;
    const float dd = __fdividef(e, e + 1.0f);
    d = bz > 20.0f ? 1.0f : dd;
    return bz > 20.0f ? z : sp;
  } else if constexpr (ACT == SR_ACT_RELU) {
    d = z > 0.f ? 1.f : 0.f;
    return fmaxf(z, 0.f);
  } else if constexpr (ACT == SR_ACT_TANH) {
    const float t = tanhf(z);
    d = 1.f - t * t;
    return t;
  } else {
    d = 1.f;
    return z;
  }
}

__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// value only (the common epilogue: no tangent rows, no stash): 2 MUFU per softplus
template <int ACT>
__device__ __forceinline__ float act_val(float z) {
  if constexpr (ACT == SR_ACT_SOFTPLUS100) {
    // softplus(beta = 100, threshold 20): log(1 + exp(100 z)) / 100, z itself above the threshold
    const float t = z * 144.26950408889634f;                       // 100 z log2(e)
    const float e = fast_ex2(fminf(t, 28.853900817779268f));       // exp(min(100 z, 20))
    const float sp = fast_lg2(1.0f + e) * 0.006931471805599453f;   // ln(2) / 100
    return t > 28.853900817779268f ? z : sp;
  } else if constexpr (ACT == SR_ACT_RELU) {
    return fmaxf(z, 0.f);
  } else if constexpr (ACT == SR_ACT_TANH) {
    return tanhf(z);
  } else {
    return z;
  }
}
// act'(z) recovered from the activation value a = act(z)
template <int ACT>
__device__ __forceinline__ float dact_from_val(float a) {
  if constexpr (ACT == SR_ACT_SOFTPLUS100) return 1.0f - fast_ex2(a * -144.26950408889634f);
  else if constexpr (ACT == SR_ACT_RELU) return a > 0.f ? 1.f : 0.f;
  else if constexpr (ACT == SR_ACT_TANH) return 1.f - a * a;
  else return 1.f;
}

// two fp32 values -> three packed bf16 pairs (element 0 in the low half = lower address)
__device__ __forceinline__ void split3x2(float x0, float x1, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
  __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  p1 = *reinterpret_cast<uint32_t*>(&h);
  const float r0 = x0 - __uint_as_float(p1 << 16), r1 = x1 - __uint_as_float(p1 & 0xffff0000u);
  h = __floats2bfloat162_rn(r0, r1);
  p2 = *reinterpret_cast<uint32_t*>(&h);
  if constexpr (kPlanes == 3) {
    const float s0 = r0 - __uint_as_float(p2 << 16), s1 = r1 - __uint_as_float(p2 & 0xffff0000u);
    h = __floats2bfloat162_rn(s0, s1);
    p3 = *reinterpret_cast<uint32_t*>(&h);
  } else {
    p3 = 0u;
  }
}

struct EpiRow {
  long long mt, row;
  int row_in_tile, lane;
  bool row_ok, is_val;
  size_t ds_ld;
};

// A reverse launch's epilogue reads the previous layer's activation tile of chunk c0 (act' is recomputed from it) only
// for columns < n; the producer stages exactly these chunks in the operand ring (tc_sweep_kernel), and both sides
// decide with this one rule.
__device__ __forceinline__ bool mul_chunk_staged(const LayerArgs& a, int c0) { return c0 < a.n && (c0 >> 5) < a.mul_KC; }

// One 32-column chunk of the accumulator (this thread: one row), layer columns [c0, c0 + 32): bias / activation /
// tangent scaling (forward) or act' multiply (reverse), then the fp32 outputs, the act' stash and the re-split bf16
// tile of the next layer.  `live` = the chunk holds GEMM columns (else only the zero padding / skip-connection columns
// of the next layer's input are produced).  `mul_stage` (reverse launches): the ring slot holding this chunk's
// activation tile (one A stage, both planes), or null when the chunk has no columns < n (act' is then unused).
template <int ACT, int CH, bool MUL, bool PF = true>
__device__ __forceinline__ void epi_chunk(const LayerArgs& a, const EpiRow& r, uint32_t (&v)[32], int c0, bool live,
                                          const __nv_bfloat16* mul_stage = nullptr) {
  float o[32];
  if (live) {
    if constexpr (MUL) {
      // reverse sweep: delta * act'(z) for the columns that continue; columns >= n (the skip part of
      // a skip layer's input gradient) pass through unscaled.  ACT is the PREVIOUS layer's activation.
      const __nv_bfloat16* mt =
          mul_stage + (size_t)(r.row_in_tile >> 3) * 64 + (r.row_in_tile & 7) * 8;   // shared memory
      const float kk = -144.26950408889634f * a.mul_inv_scale;   // -100 log2(e) / scale
      // optional fp32 act'(z) of the previous layer's VALUE rows (written by its forward launch as `dstash`, row
      // pitch pad256(n)); only chunks with columns < n use act', the skip columns of a skip layer's input have none.
      // Rows past M read row 0's entries (discarded below)
      const long long srow = r.row_ok ? (CH == 4 ? (r.row & ~3LL) : r.row) : 0;
      const float* stash = a.dstash == nullptr || c0 >= a.n ? nullptr : a.dstash + (size_t)srow * r.ds_ld + c0;
      const bool use_stash = (ACT == SR_ACT_SOFTPLUS100) && stash != nullptr;
      // The activation tile comes from shared memory (staged by the producer's bulk copy under the MMAs).  The fp32
      // stash of the training sweeps stays a global load, outside the ring: it is row-major with pitch ds_ld, so a
      // chunk of it is 128 strided 128-byte pieces, not one contiguous bulk copy.  Without a staged tile (no columns
      // < n) act' is not used: zeros.
      // PF: all operands of the chunk first (8 x 16 B of activation tiles, 8 x 16 B of stash), 16 loads in flight
      // per thread; PF = false requests them per group of 8 columns (fewer registers)
      const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
      uint4 q0[PF ? 4 : 1], q1[PF ? 4 : 1];
      float st[PF ? 32 : 1];
      if constexpr (PF) {
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          q0[g] = mul_stage ? *reinterpret_cast<const uint4*>(mt + (size_t)g * (BM * 8)) : zero4;
          q1[g] = mul_stage ? *reinterpret_cast<const uint4*>(mt + (size_t)g * (BM * 8) + A_PLANE) : zero4;
        }
        if (use_stash) {
#pragma unroll
          for (int j4 = 0; j4 < 8; ++j4) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(stash) + j4);
            st[4 * j4] = t.x; st[4 * j4 + 1] = t.y; st[4 * j4 + 2] = t.z; st[4 * j4 + 3] = t.w;
          }
        }
      }
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        uint4 a0, a1;
        float sg[8];
        if constexpr (PF) {
          a0 = q0[g]; a1 = q1[g];
        } else {
          a0 = mul_stage ? *reinterpret_cast<const uint4*>(mt + (size_t)g * (BM * 8)) : zero4;
          a1 = mul_stage ? *reinterpret_cast<const uint4*>(mt + (size_t)g * (BM * 8) + A_PLANE) : zero4;
          if (use_stash) {
            const float4 t0 = __ldg(reinterpret_cast<const float4*>(stash) + 2 * g);
            const float4 t1 = __ldg(reinterpret_cast<const float4*>(stash) + 2 * g + 1);
            sg[0] = t0.x; sg[1] = t0.y; sg[2] = t0.z; sg[3] = t0.w; sg[4] = t1.x; sg[5] = t1.y; sg[6] = t1.z; sg[7] = t1.w;
          }
        }
        const uint32_t w0[4] = {a0.x, a0.y, a0.z, a0.w}, w1[4] = {a1.x, a1.y, a1.z, a1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int j = g * 8 + e;
          const uint32_t h0 = w0[e >> 1], h1 = w1[e >> 1];
          const float as = (e & 1) ? __uint_as_float(h0 & 0xffff0000u) + __uint_as_float(h1 & 0xffff0000u)
                                   : __uint_as_float(h0 << 16) + __uint_as_float(h1 << 16);
          float val = __uint_as_float(v[j]);
          if constexpr (CH == 1) {
            float d;
            if constexpr (ACT == SR_ACT_SOFTPLUS100) {
              // training: act'(z) kept in fp32 by the forward sweep (recomputing it from the 16-bit-mantissa
              // activation tiles costs 100 x 2^-17 relative on 1 - act'); the tracer recomputes (no stash traffic)
              d = use_stash ? (PF ? st[PF ? j : 0] : sg[e]) : 1.0f - fast_ex2(kk * as);
            } else if constexpr (ACT == SR_ACT_RELU) d = as > 0.f ? 1.f : 0.f;
            else d = 1.f;
            if (c0 + j < a.n) val = r.row_ok ? val * d : 0.f;
          } else {
            // Reverse sweep over forward-mode rows (value + 3 tangents per point; training: the cotangents of
            // f AND of grad f / of the offset AND of its Jacobian travel together).  With a = act(z) the stored
            // value-row activation and t_c = act'(z) u_c the stored tangent rows:
            //   tangent rows:  u_bar_c = act'(z) t_bar_c
            //   value row   :  z_bar   = act'(z) a_bar + act''(z) sum_c t_bar_c u_c
            // and act'' u_c = 100 (1 - act') t_c for softplus(beta = 100), 0 for ReLU -- no division by act'.
            float d;
            if constexpr (ACT == SR_ACT_SOFTPLUS100) {
              if (use_stash) d = PF ? st[PF ? j : 0] : sg[e];   // the four rows of a point read the value row's stash entry
              else d = 1.0f - fast_ex2(kk * __shfl_sync(0xffffffffu, as, r.lane & ~3));
            } else if constexpr (ACT == SR_ACT_RELU) {
              d = __shfl_sync(0xffffffffu, as, r.lane & ~3) > 0.f ? 1.f : 0.f;
            } else d = 1.f;
            float cross = 0.f;
            if constexpr (ACT == SR_ACT_SOFTPLUS100) {
              // sum of t_bar_c * t_c over the three tangent lanes of the point (butterfly inside the lane quad)
              float prod = r.is_val ? 0.f : val * (as * a.mul_inv_scale);
              prod += __shfl_xor_sync(0xffffffffu, prod, 1);
              prod += __shfl_xor_sync(0xffffffffu, prod, 2);
              cross = prod;
            }
            if (c0 + j < a.n) {
              float o4 = val * d;
              if constexpr (ACT == SR_ACT_SOFTPLUS100) { if (r.is_val) o4 += 100.0f * (1.0f - d) * cross; }
              val = r.row_ok ? o4 : 0.f;
            }
          }
          o[j] = val * a.scale;
        }
      }
    } else {
#pragma unroll
      for (int j4 = 0; j4 < 8; ++j4) {
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(a.bias + c0) + j4);
        const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = j4 * 4 + jj;
          const float acc = __uint_as_float(v[j]);
          float val;
          if constexpr (CH == 1) {
            val = act_val<ACT>(acc + bb[jj]);
          } else {
            float d = 1.f;
            val = act_fn<ACT>(acc + bb[jj], d);                          // meaningful on value rows
            const float dv = __shfl_sync(0xffffffffu, d, r.lane & ~3);  // act'(z) of the value row
            if (!r.is_val) { val = dv * acc; }
            v[j] = __float_as_uint(d);
          }
          o[j] = val * a.scale;
        }
      }
      if (a.dstash != nullptr && r.is_val && r.row_ok) {
        if constexpr (CH == 1) {   // rarely used output: act' recomputed from the activation values
          const float inv = 1.0f / a.scale;
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(dact_from_val<ACT>(o[j] * inv));
        }
        float4* dd = reinterpret_cast<float4*>(a.dstash + (size_t)r.row * r.ds_ld + c0);
#pragma unroll
        for (int j4 = 0; j4 < 8; ++j4)
          dd[j4] = make_float4(__uint_as_float(v[4 * j4]), __uint_as_float(v[4 * j4 + 1]),
                               __uint_as_float(v[4 * j4 + 2]), __uint_as_float(v[4 * j4 + 3]));
      }
    }
    if (a.out != nullptr && r.row_ok && c0 < a.out_col0 + a.out_n && c0 + 32 > a.out_col0) {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int c = c0 + j - a.out_col0;
        if (c >= 0 && c < a.out_n) a.out[(size_t)r.row * a.out_ld + c] = o[j];
      }
    }
  }
  if (a.A_next == nullptr) return;
  const int kcn = c0 >> 5;  // next layer's k chunk
  if (kcn >= a.KCn) return;
  if (!live || c0 + 32 > a.n) {  // zero padding / skip-connection columns (uniform branch)
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int c = c0 + j;
      if (!live || c >= a.n) {
        float val = 0.f;
        if (a.skip_src != nullptr && c >= a.n && c < a.n + a.skip_n && r.row_ok)
          val = a.skip_src[(size_t)r.row * a.skip_ld + (c - a.n)] * a.scale;
        o[j] = val;
      }
    }
  }
  __nv_bfloat16* base = a.A_next + a_tile_off(r.mt, kcn, a.KCn, 0) + (size_t)(r.row_in_tile >> 3) * 64 +
                        (r.row_in_tile & 7) * 8;
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    uint4 q1, q2, q3;
    split3x2(o[g * 8 + 0], o[g * 8 + 1], q1.x, q2.x, q3.x);
    split3x2(o[g * 8 + 2], o[g * 8 + 3], q1.y, q2.y, q3.y);
    split3x2(o[g * 8 + 4], o[g * 8 + 5], q1.z, q2.z, q3.z);
    split3x2(o[g * 8 + 6], o[g * 8 + 7], q1.w, q2.w, q3.w);
    __nv_bfloat16* dst = base + (size_t)g * (BM * 8);
    *reinterpret_cast<uint4*>(dst) = q1;
    *reinterpret_cast<uint4*>(dst + A_PLANE) = q2;
    if constexpr (kPlanes == 3) *reinterpret_cast<uint4*>(dst + 2 * A_PLANE) = q3;
  }
}


// ---- the layer kernel: one layer per launch ------------------------------------------------------------------------
// The name tc_sweep_kernel is kept: the benchmark's roofline label names it and tools/prof_train_kernels.py matches it.
// Persistent CTAs, at most one per SM: CTA c owns the row tiles {c, c + grid, ...} and runs every n-tile of each.
// The column tile is TBN = 256, or 64 for narrow layers (N <= 64: the SDF's last layer, the translator's output, the
// input gradient of a reverse sweep): a 64-column tile streams a quarter of the weight bytes per k chunk and issues
// n64 MMAs, where a 256-column tile would multiply zero-padded weight rows.
//
// Roles (3 warpgroups): warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = rows [0, 64) and [64, 128) of
// the 128 x TBN output tile: wgmma m64nTBNk16 with fp32 accumulators in registers (TBN / 2 per thread), then the
// epilogue of the same rows.  The accumulator goes through shared memory (up to 128 columns at a time) so that each
// epilogue thread owns one row and 32 consecutive columns per chunk: the four rows of a point (value + 3 tangents)
// sit in four consecutive lanes.
constexpr int kConsumerWGs = 2;
constexpr int kThreads = 128 * (1 + kConsumerWGs);
constexpr int kEpiWarps = 4 * kConsumerWGs;
constexpr int STG_LD = 132;                 // staging row pitch (floats): conflict-free float4 row reads
constexpr int STG_FLOATS = 64 * STG_LD;     // per consumer warpgroup: 64 rows x 128 columns
template <int TBN>
constexpr uint32_t w_stage_bytes() { return (uint32_t)kPlanes * TBN * BK * 2; }   // 2 planes: 32 KB (TBN 256), 8 KB (64)
// Ring depth.  The narrow tile's stages are half the size (24 KB) and its MMAs short, so its launches are bound by
// the A stream; twice the stages keep twice the bytes in flight in the same shared memory as the wide tile's ring.
template <int TBN>
constexpr int ring_stages() { return TBN == BN ? STAGES : 2 * STAGES; }
template <int TBN>
constexpr size_t smem_bytes() {
  return (size_t)ring_stages<TBN>() * (A_STAGE_BYTES + w_stage_bytes<TBN>()) + (size_t)kConsumerWGs * STG_FLOATS * 4 + 256;
}
static_assert(smem_bytes<BN>() <= 227 * 1024 && smem_bytes<BN_NARROW>() <= 227 * 1024, "shared memory of one H100 block");
static_assert(2 * ring_stages<BN_NARROW>() * sizeof(uint64_t) <= 256, "full + empty barriers fit their 256 bytes");

// Epilogue stages of a reverse launch.  The epilogue runs an n-tile in passes of PASS columns (128, or 64 on the narrow
// tile); in each pass the warps with (wq >> 1) = q take columns [q PASS / 2, (q + 1) PASS / 2), chunk i = 0 .. WCH - 1
// in turn, both halves at the same time.  The producer stages the previous layer's activation tile of each chunk
// (16 KB, both planes: exactly one A stage) in the ring, in that order: on the wide tile one stage carries chunk i of
// both halves, half 0's in the slot's A part and half 1's in its (32 KB) W part; on the narrow tile (8 KB W part) a
// stage carries one chunk, half 0's then half 1's.  kEpiHalves = halves per stage.
template <int TBN>
constexpr int kEpiHalves = TBN == BN ? 2 : 1;
static_assert(w_stage_bytes<BN>() >= A_STAGE_BYTES, "the wide tile's W stage holds one activation chunk");
template <int TBN>
__device__ __forceinline__ int epi_chunk_col(int nt, int h, int q, int i) {
  constexpr int PASS = TBN < 128 ? TBN : 128;
  return nt * TBN + h * PASS + q * (PASS / 2) + 32 * i;
}
// where half q's chunk of the stage in ring slot `slot` lands (q0 = the stage's first half)
template <int TBN>
__device__ __forceinline__ __nv_bfloat16* epi_stage_dst(__nv_bfloat16* sA, __nv_bfloat16* sW, int slot, int q, int q0) {
  return q == q0 ? sA + (size_t)slot * A_STAGE : sW + (size_t)slot * (w_stage_bytes<TBN>() / 2);
}

// One k chunk of this warpgroup's 64 x TBN tile: the split-bf16 product terms, plane pairs smallest contributions
// first -- 2 planes: (a0,w1) (a1,w0) (a0,w0); 3 planes: (a0,w2) (a2,w0) (a1,w1) (a0,w1) (a1,w0) (a0,w0).
// abase = this warpgroup's first row group of the A stage, wbase = the W stage.
template <int TBN, bool FIRST>
__device__ __forceinline__ void mma_chunk(float (&acc)[TBN / 2], uint32_t abase, uint32_t wbase) {
  constexpr int kTerms = kPlanes == 2 ? 3 : 6;
  const int pa[6] = {0, 1, 0, 2, 1, 0}, pw[6] = {1, 0, 0, 0, 1, 0};
  const int pa3[6] = {0, 2, 1, 0, 1, 0}, pw3[6] = {2, 0, 1, 1, 0, 0};
#pragma unroll
  for (int q = 0; q < kTerms; ++q) {
#pragma unroll
    for (int jj = 0; jj < BK / 16; ++jj) {
      // K = 16 per MMA = two 8-wide core matrices: advance two LBO steps per jj
      const int qa = kPlanes == 2 ? pa[q] : pa3[q], qw = kPlanes == 2 ? pw[q] : pw3[q];
      const uint64_t ad = make_desc(abase + qa * (A_PLANE * 2) + jj * 2 * (BM * 16), BM * 16, 128);
      const uint64_t bd = make_desc(wbase + qw * (TBN * BK * 2) + jj * 2 * (TBN * 16), TBN * 16, 128);
      const bool first = FIRST && q == 0 && jj == 0;
      if constexpr (TBN == BN) {
        if (first) wgmma_m64n256k16<0, 0, true>(acc, ad, bd);
        else wgmma_m64n256k16<0, 0, false>(acc, ad, bd);
      } else {
        static_assert(TBN == BN_NARROW, "column tile");
        if (first) wgmma_m64n64k16<0, 0, true>(acc, ad, bd);
        else wgmma_m64n64k16<0, 0, false>(acc, ad, bd);
      }
    }
  }
}

// <ACT, CH, MUL, TBN>: the layer's activation (a reverse launch: the PREVIOUS layer's), rows per point, reverse mode,
// column tile
template <int ACT, int CH, bool MUL, int TBN>
__global__ void __launch_bounds__(kThreads, 1) tc_sweep_kernel(const __grid_constant__ LayerArgs a) {
  constexpr uint32_t W_STAGE_BYTES = w_stage_bytes<TBN>();
  constexpr int NS = ring_stages<TBN>();
  constexpr int W_STAGE = W_STAGE_BYTES / 2;   // elements
  extern __shared__ __align__(1024) unsigned char smem[];
  __nv_bfloat16* sA = reinterpret_cast<__nv_bfloat16*>(smem);
  __nv_bfloat16* sW = reinterpret_cast<__nv_bfloat16*>(smem + (size_t)NS * A_STAGE_BYTES);
  float* stg = reinterpret_cast<float*>(smem + (size_t)NS * (A_STAGE_BYTES + W_STAGE_BYTES));
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg + kConsumerWGs * STG_FLOATS);
  uint64_t* full = bars;                    // [NS] operands of the stage landed (producer expect_tx)
  uint64_t* empty = bars + NS;              // [NS] the MMAs of every consumer warp have read the stage

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    for (int i = 0; i < NS; ++i) { sr_mbar_init(&full[i], 1); sr_mbar_init(&empty[i], kEpiWarps); }
    sr_fence_barrier_init();
  }
  __syncthreads();
  long long Mrows = a.M;
  int MTe = a.MT;
  if (a.m_dev != nullptr) {
    const long long md = (long long)(*a.m_dev);
    Mrows = md < a.M ? md : a.M;
    MTe = (int)((Mrows + BM - 1) / BM);
  }
  const int cta = blockIdx.x, ncta = gridDim.x;
  const int J = cta < MTe ? (MTe - cta + ncta - 1) / ncta : 0;   // row tiles of this CTA

  // 384 threads at one block per SM start with 168 registers each; the producer warpgroup hands most of its share to
  // the consumers (128 accumulators + epilogue state per thread): 128 x 40 + 256 x 232 <= 65 536
  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int slot = 0;
      uint32_t phase = 0;
      for (int j = 0; j < J; ++j) {
        const long long mt = (long long)cta + (long long)j * ncta;
        for (int nt = 0; nt < a.NT; ++nt) {
          for (int kc = 0; kc < a.KC; ++kc) {
            sr_mbar_wait(&empty[slot], phase ^ 1u);
            sr_mbar_arrive_expect_tx(&full[slot], A_STAGE_BYTES + W_STAGE_BYTES);
            sr_bulk_g2s(sW + (size_t)slot * W_STAGE, a.W + w_tile_off(TBN, nt, kc, a.KC, 0), W_STAGE_BYTES, &full[slot]);
            sr_bulk_g2s(sA + (size_t)slot * A_STAGE, a.A + a_tile_off(mt, kc, a.KC, 0), A_STAGE_BYTES, &full[slot]);
            if (++slot == NS) { slot = 0; phase ^= 1u; }
          }
          if constexpr (MUL) {
            // epilogue stages: the previous layer's activation tiles of the chunks this n-tile's epilogue reads, in
            // its consumption order (kEpiHalves)
            constexpr int PASS = TBN < 128 ? TBN : 128, WCH = PASS / 64, EH = kEpiHalves<TBN>;
            for (int h = 0; h < TBN / PASS; ++h) {
              for (int i = 0; i < WCH; ++i) {
                for (int q0 = 0; q0 < 2; q0 += EH) {
                  uint32_t bytes = 0;
                  for (int q = q0; q < q0 + EH; ++q)
                    if (mul_chunk_staged(a, epi_chunk_col<TBN>(nt, h, q, i))) bytes += A_STAGE_BYTES;
                  if (bytes == 0) continue;
                  sr_mbar_wait(&empty[slot], phase ^ 1u);
                  sr_mbar_arrive_expect_tx(&full[slot], bytes);
                  for (int q = q0; q < q0 + EH; ++q) {
                    const int c0 = epi_chunk_col<TBN>(nt, h, q, i);
                    if (mul_chunk_staged(a, c0))
                      sr_bulk_g2s(epi_stage_dst<TBN>(sA, sW, slot, q, q0),
                                  a.mul_tiles + a_tile_off(mt, c0 >> 5, a.mul_KC, 0), A_STAGE_BYTES, &full[slot]);
                  }
                  if (++slot == NS) { slot = 0; phase ^= 1u; }
                }
              }
            }
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue (warpgroups 1, 2)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;                  // rows [64 cw, 64 cw + 64) of the row tile
    const int wq = warp & 3;                // warp in the warpgroup
    float* st = stg + cw * STG_FLOATS;
    float acc[TBN / 2];
    EpiRow r;
    r.row_in_tile = cw * 64 + (wq & 1) * 32 + lane;
    r.lane = lane;
    r.is_val = (CH == 1) || ((lane & 3) == 0);
    // act' stash pitch (either column tile): a forward launch writes pad256(N); a reverse launch reads the previous
    // layer's stash, whose width is this launch's n (N = n + d_in for a skip layer, which may cross a multiple of 256)
    r.ds_ld = (size_t)(((MUL ? a.n : a.n_gemm) + BN - 1) / BN) * BN;
    int slot = 0;
    uint32_t phase = 0;
    for (int j = 0; j < J; ++j) {
      r.mt = (long long)cta + (long long)j * ncta;
      r.row = r.mt * BM + r.row_in_tile;
      r.row_ok = r.row < Mrows;
      for (int nt = 0; nt < a.NT; ++nt) {
        // the first k chunk overwrites the accumulator (it is dead from here back to the previous epilogue)
        sr_mbar_wait(&full[slot], phase);
        wgmma_fence();
        mma_chunk<TBN, true>(acc, sr_smem_u32(sA + (size_t)slot * A_STAGE) + cw * 8 * 128,
                             sr_smem_u32(sW + (size_t)slot * W_STAGE));
        wgmma_commit();
        int prev = slot;
        if (++slot == NS) { slot = 0; phase ^= 1u; }
        for (int kc = 1; kc < a.KC; ++kc) {
          sr_mbar_wait(&full[slot], phase);
          wgmma_fence();
          mma_chunk<TBN, false>(acc, sr_smem_u32(sA + (size_t)slot * A_STAGE) + cw * 8 * 128,
                                sr_smem_u32(sW + (size_t)slot * W_STAGE));
          wgmma_commit();
          wgmma_wait<1>();   // the previous stage's MMAs are complete: release it
          if (lane == 0) sr_mbar_arrive(&empty[prev]);
          prev = slot;
          if (++slot == NS) { slot = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        if (lane == 0) sr_mbar_arrive(&empty[prev]);
        // epilogue: PASS accumulator columns per pass through the staging buffer; warp wq handles rows
        // 32 (wq & 1) + lane and the PASS / 2 columns (PASS / 2) (wq >> 1) of each pass (PASS / 64 32-column chunks)
        constexpr int PASS = TBN < 128 ? TBN : 128, FRAGS = PASS / 8, WCH = PASS / 64;
#pragma unroll
        for (int h = 0; h < TBN / PASS; ++h) {
          const int fr = 16 * wq + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
          for (int i = 0; i < FRAGS; ++i) {
            *reinterpret_cast<float2*>(st + fr * STG_LD + 8 * i + fc) =
                make_float2(acc[4 * (FRAGS * h + i)], acc[4 * (FRAGS * h + i) + 1]);
            *reinterpret_cast<float2*>(st + (fr + 8) * STG_LD + 8 * i + fc) =
                make_float2(acc[4 * (FRAGS * h + i) + 2], acc[4 * (FRAGS * h + i) + 3]);
          }
          warpgroup_sync(1 + cw);
          const float* srow = st + ((wq & 1) * 32 + lane) * STG_LD + (wq >> 1) * (PASS / 2);
          auto chunk = [&](int i, int c0, const __nv_bfloat16* mul_stage) {
            uint32_t v[32];
#pragma unroll
            for (int j4 = 0; j4 < 8; ++j4) {
              const float4 t = reinterpret_cast<const float4*>(srow + 32 * i)[j4];
              v[4 * j4] = __float_as_uint(t.x); v[4 * j4 + 1] = __float_as_uint(t.y);
              v[4 * j4 + 2] = __float_as_uint(t.z); v[4 * j4 + 3] = __float_as_uint(t.w);
            }
            epi_chunk<ACT, CH, MUL>(a, r, v, c0, c0 < a.n_gemm, mul_stage);
          };
          if constexpr (!MUL) {
            for (int i = 0; i < WCH; ++i) chunk(i, nt * TBN + h * PASS + (wq >> 1) * (PASS / 2) + 32 * i, nullptr);
          } else {
            // The pass's epilogue stages in ring order (kEpiHalves).  Every warp of both warpgroups waits for every
            // stage and releases it in that order, reading only its own half's chunk (on the narrow tile a warp
            // releases the other half's stage unread): the producer refills a slot only after all kEpiWarps warps
            // released it.  No deadlock: a warp's wait for stage s depends only on releases of stages <= s - NS,
            // and each warp releases stage s after its wait for s and at most its own chunk's work, never after a
            // later stage, so the releases of the earliest unreleased stage always complete.  Waiting before a
            // release also keeps a warp that skips a stage from arriving while the slot's previous use is open.
            constexpr int EH = kEpiHalves<TBN>;
            const int qm = wq >> 1;
            for (int i = 0; i < WCH; ++i) {
              for (int q0 = 0; q0 < 2; q0 += EH) {
                bool any = false;
                for (int q = q0; q < q0 + EH; ++q) any |= mul_chunk_staged(a, epi_chunk_col<TBN>(nt, h, q, i));
                const bool mine = qm >= q0 && qm < q0 + EH;
                const int c0 = epi_chunk_col<TBN>(nt, h, qm, i);
                const __nv_bfloat16* mul_stage = nullptr;
                if (any) {
                  sr_mbar_wait(&full[slot], phase);
                  if (mul_chunk_staged(a, c0)) mul_stage = epi_stage_dst<TBN>(sA, sW, slot, qm, q0);
                }
                if (mine) chunk(i, c0, mul_stage);
                if (any) {
                  __syncwarp();
                  if (lane == 0) sr_mbar_arrive(&empty[slot]);
                  if (++slot == NS) { slot = 0; phase ^= 1u; }
                }
              }
            }
          }
          warpgroup_sync(1 + cw);
        }
      }
    }
  }
}

// ---- packing kernels -------------------------------------------------------------------------
// fp32 row-major [M][K] (ld) -> tiled split-bf16 activations with KC = ceil(Kpad/32) chunks
__global__ void pack_rows_kernel(const float* __restrict__ src, long long M, int K, int ld,
                                 __nv_bfloat16* __restrict__ dst, int KC, long long MT,
                                 const int* __restrict__ m_dev) {
  if (m_dev != nullptr) {
    const long long md = *m_dev;
    M = md < M ? md : M;
    MT = (M + BM - 1) / BM;
  }
  const long long total = MT * BM * (long long)KC * 4;  // one thread per (row, k8 group)
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(idx % BM);
    const long long rest = idx / BM;
    const int g = (int)(rest % (KC * 4));
    const long long mt = rest / (KC * 4);
    const long long row = mt * BM + r;
    const int kc = g >> 2, k8 = g & 3;
    __align__(16) __nv_bfloat16 p1[8], p2[8], p3[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = kc * 32 + k8 * 8 + e;
      const float x = (row < M && k < K) ? src[(size_t)row * ld + k] : 0.f;
      split3(x, p1[e], p2[e], p3[e]);
    }
    const size_t off = (size_t)k8 * (BM * 8) + (size_t)(r >> 3) * 64 + (r & 7) * 8;
    *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, KC, 0) + off) = *reinterpret_cast<uint4*>(p1);
    *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, KC, 1) + off) = *reinterpret_cast<uint4*>(p2);
    if constexpr (kPlanes == 3)
      *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, KC, kPlanes - 1) + off) = *reinterpret_cast<uint4*>(p3);
  }
}

// k chunks [kc0, KCn) of a layer's next-layer tiles that lie past its last column tile, which the layer kernel's
// epilogue never reaches: a skip layer's input n + skip_n can be wider than pad256(n).  scale * skip_src in columns
// [n, n + skip_n), zero elsewhere and in rows past the (device-side) row count, as the epilogue writes them.
__global__ void pack_skip_tail_kernel(const float* __restrict__ skip_src, int skip_ld, int n, int skip_n, float scale,
                                      long long M, int kc0, int KCn, __nv_bfloat16* __restrict__ dst,
                                      const int* __restrict__ m_dev) {
  if (m_dev != nullptr) {
    const long long md = *m_dev;
    M = md < M ? md : M;
  }
  const long long MT = (M + BM - 1) / BM;
  const int nkc = KCn - kc0;
  const long long total = MT * BM * (long long)nkc * 4;  // one thread per (row, k8 group)
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(idx % BM);
    const long long rest = idx / BM;
    const int g = (int)(rest % (nkc * 4));
    const long long mt = rest / (nkc * 4);
    const long long row = mt * BM + r;
    const int kc = kc0 + (g >> 2), k8 = g & 3;
    __align__(16) __nv_bfloat16 p1[8], p2[8], p3[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = kc * 32 + k8 * 8 + e;
      const float x = (skip_src != nullptr && row < M && c >= n && c < n + skip_n)
                          ? skip_src[(size_t)row * skip_ld + (c - n)] * scale : 0.f;
      split3(x, p1[e], p2[e], p3[e]);
    }
    const size_t off = (size_t)k8 * (BM * 8) + (size_t)(r >> 3) * 64 + (r & 7) * 8;
    *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, KCn, 0) + off) = *reinterpret_cast<uint4*>(p1);
    *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, KCn, 1) + off) = *reinterpret_cast<uint4*>(p2);
    if constexpr (kPlanes == 3)
      *reinterpret_cast<uint4*>(dst + a_tile_off(mt, kc, KCn, kPlanes - 1) + off) = *reinterpret_cast<uint4*>(p3);
  }
}

// effective weights, fp32 row-major [N][K] (ld) -> tiled split-bf16 [NT][KC][planes][bn x 32], bn = tile_n(N)
__global__ void pack_weights_kernel(const float* __restrict__ w, int N, int K, int ld,
                                    __nv_bfloat16* __restrict__ dst, int NT, int KC) {
  const int bn = tile_n(N);
  const long long total = (long long)NT * bn * KC * 4;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(idx % bn);
    const long long rest = idx / bn;
    const int g = (int)(rest % (KC * 4));
    const int nt = (int)(rest / (KC * 4));
    const int n = nt * bn + r;
    const int kc = g >> 2, k8 = g & 3;
    __align__(16) __nv_bfloat16 p1[8], p2[8], p3[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = kc * 32 + k8 * 8 + e;
      const float x = (n < N && k < K) ? w[(size_t)n * ld + k] : 0.f;
      split3(x, p1[e], p2[e], p3[e]);
    }
    const size_t off = (size_t)k8 * (bn * 8) + (size_t)(r >> 3) * 64 + (r & 7) * 8;
    *reinterpret_cast<uint4*>(dst + w_tile_off(bn, nt, kc, KC, 0) + off) = *reinterpret_cast<uint4*>(p1);
    *reinterpret_cast<uint4*>(dst + w_tile_off(bn, nt, kc, KC, 1) + off) = *reinterpret_cast<uint4*>(p2);
    if constexpr (kPlanes == 3)
      *reinterpret_cast<uint4*>(dst + w_tile_off(bn, nt, kc, KC, kPlanes - 1) + off) = *reinterpret_cast<uint4*>(p3);
  }
}

// Embedded network input, fp32 row-major [P*ch][ld]: PE(p) (+ cond[b]) for value rows and
// d/dp_t of it for tangent rows (model/Embedder.py:11-32).  One thread per element (coalesced).
struct EmbedArgs {
  const float* pts;
  long long P;
  int multires;
  float pe_w[16];
  int ch;
  const float* conds;
  const long long* batch_inds;
  long long pts_per_frame;
  int condlen;
  float* out;
  int ld;
  const int* index;   // optional active list: row i embeds point index[i]
  const int* m_dev;   // optional device-side count of active points
};
__global__ void embed_kernel(const __grid_constant__ EmbedArgs a) {
  long long np = a.P;
  if (a.m_dev != nullptr) { const long long md = *a.m_dev; np = md < np ? md : np; }
  const long long total = np * a.ch * (long long)a.ld;
  const int pe_dim = 3 + 6 * a.multires;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(idx % a.ld);
    const long long row = idx / a.ld;
    const long long pi = row / a.ch;
    const long long p = a.index ? (long long)a.index[pi] : pi;
    const int t = (int)(row % a.ch);  // 0 = value, 1..3 = d/dp_{t-1}
    float v = 0.f;
    if (k < 3) {
      v = t == 0 ? a.pts[p * 3 + k] : (t - 1 == k ? 1.f : 0.f);
    } else if (k < pe_dim) {
      const int b = (k - 3) / 6, w6 = (k - 3) % 6, j = w6 % 3;
      const bool is_cos = w6 >= 3;
      if (t == 0 || t - 1 == j) {
        const float freq = (float)(1 << b);
        float sn, cs;
        sincosf(a.pts[p * 3 + j] * freq, &sn, &cs);
        const float w = a.pe_w[b];
        if (t == 0) v = w * (is_cos ? cs : sn);
        else v = is_cos ? -(w * freq) * sn : (w * freq) * cs;
      }
    } else if (k < pe_dim + a.condlen) {
      if (t == 0) {
        const long long bi = a.batch_inds ? a.batch_inds[p] : (a.pts_per_frame > 0 ? p / a.pts_per_frame : 0);
        v = a.conds[bi * a.condlen + (k - pe_dim)];
      }
    }
    a.out[idx] = v;
  }
}

// Backward of embed_kernel w.r.t. the points: gx [P*ch][ld] cotangent rows -> gp [P][3].  Value row: d PE / d p; tangent
// rows (ch = 4): the tangent entries themselves depend on p (second derivative of the encoding).  gk (ch = 1, or null):
// a second cotangent of the same input, [P][gk_ld] -- a skip layer's part of the reverse sweep.  One thread per point.
__global__ void embed_bwd_kernel(const float* __restrict__ pts, long long P, int multires, const float* __restrict__ gx,
                                 int ld, int ch, const float* __restrict__ gk, int gk_ld, float* __restrict__ gp,
                                 float pw0, float pw1, float pw2, float pw3, float pw4, float pw5, float pw6, float pw7) {
  const float pw[8] = {pw0, pw1, pw2, pw3, pw4, pw5, pw6, pw7};
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
    const float* gv = gx + (size_t)p * ch * ld;
    const float* gs = gk != nullptr ? gk + (size_t)p * gk_ld : nullptr;
    float out[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const float x = pts[p * 3 + j];
      float acc = gv[j] + (gs ? gs[j] : 0.f);
      const float* gt = ch == 4 ? gv + (size_t)(1 + j) * ld : nullptr;   // tangent row d/dp_j: only column j is non-zero
      float freq = 1.0f;
      for (int b = 0; b < multires; ++b, freq *= 2.0f) {
        float sn, cs;
        sincosf(x * freq, &sn, &cs);
        const float w = pw[b] * freq;
        const int ks = 3 + 6 * b + j, kc = ks + 3;
        const float gsn = gv[ks] + (gs ? gs[ks] : 0.f), gcs = gv[kc] + (gs ? gs[kc] : 0.f);
        acc += w * (cs * gsn - sn * gcs);
        if (gt) acc -= w * freq * (sn * gt[ks] + cs * gt[kc]);
      }
      out[j] = acc;
    }
    gp[p * 3] = out[0]; gp[p * 3 + 1] = out[1]; gp[p * 3 + 2] = out[2];
  }
}

}  // namespace sr_tc

extern "C" {

int sr_tc_embed_backward(const float* pts, int64_t P, int multires, const float* pe_w, int ch, const float* gx, int ld,
                         const float* gk, int gk_ld, float* gp, cudaStream_t s) {
  if (!pts || !gx || !gp || !pe_w || P <= 0 || (ch != 1 && ch != 4) || multires < 0 || multires > 8 ||
      ld < 3 + 6 * multires || (gk && (ch != 1 || gk_ld < 3 + 6 * multires)))
    return SR_EINVAL;
  float w[8];
  for (int i = 0; i < 8; ++i) w[i] = i < multires ? pe_w[i] : 0.f;
  sr_tc::embed_bwd_kernel<<<sr_grid_for(P, 256, 8), 256, 0, s>>>(pts, P, multires, gx, ld, ch, gk, gk_ld, gp, w[0], w[1],
                                                                  w[2], w[3], w[4], w[5], w[6], w[7]);
  return sr_launch_status();
}

int sr_tc_embed(const float* pts, int64_t P, int multires, const float* pe_w, int ch,
                const float* conds, const int64_t* batch_inds, int64_t pts_per_frame, int condlen,
                float* out, int ld, const int32_t* index, const int32_t* m_dev, cudaStream_t s) {
  if (!pts || !out || !pe_w || P <= 0 || (ch != 1 && ch != 4) || multires < 0 || multires > 16) return SR_EINVAL;
  if (ld < 3 + 6 * multires + condlen || (condlen > 0 && !conds)) return SR_EINVAL;
  sr_tc::EmbedArgs a;
  a.pts = pts; a.P = P; a.multires = multires; a.ch = ch; a.conds = conds;
  a.batch_inds = (const long long*)batch_inds; a.pts_per_frame = pts_per_frame; a.condlen = condlen;
  a.out = out; a.ld = ld; a.index = index; a.m_dev = m_dev;
  for (int i = 0; i < 16; ++i) a.pe_w[i] = i < multires ? pe_w[i] : 0.f;
  const long long total = P * ch * (long long)ld;
  sr_tc::embed_kernel<<<sr_grid_for(total, 256, 8), 256, 0, s>>>(a);
  return sr_launch_status();
}

int64_t sr_tc_act_bytes(int64_t M, int K) {
  const int64_t MT = (M + sr_tc::BM - 1) / sr_tc::BM, KC = (K + 31) / 32;
  return MT * KC * sr_tc::kPlanes * sr_tc::A_PLANE * 2;
}
int64_t sr_tc_weight_bytes(int N, int K) {
  const int64_t bn = sr_tc::tile_n(N), NT = (N + bn - 1) / bn, KC = (K + 31) / 32;
  return NT * KC * sr_tc::kPlanes * bn * sr_tc::BK * 2;
}

int sr_tc_pack_rows(const float* src, int64_t M, int K, int ld, void* dst, const int32_t* m_dev,
                    cudaStream_t s) {
  if (!src || !dst || M <= 0 || K <= 0 || ld < K) return SR_EINVAL;
  const long long MT = (M + sr_tc::BM - 1) / sr_tc::BM;
  const int KC = (K + 31) / 32;
  const long long total = MT * sr_tc::BM * KC * 4;
  sr_tc::pack_rows_kernel<<<sr_grid_for(total, 256, 8), 256, 0, s>>>(src, M, K, ld, (__nv_bfloat16*)dst, KC, MT, m_dev);
  return sr_launch_status();
}

int sr_tc_pack_weights(const float* w, int N, int K, int ld, void* dst, cudaStream_t s) {
  if (!w || !dst || N <= 0 || K <= 0 || ld < K) return SR_EINVAL;
  const int bn = sr_tc::tile_n(N), NT = (N + bn - 1) / bn, KC = (K + 31) / 32;
  const long long total = (long long)NT * bn * KC * 4;
  sr_tc::pack_weights_kernel<<<sr_grid_for(total, 256, 8), 256, 0, s>>>(w, N, K, ld, (__nv_bfloat16*)dst, NT, KC);
  return sr_launch_status();
}

// picks the instantiation for (activation, mode, ch) and launches one CTA per row tile, at most one per SM; when the
// next layer's input is wider than pad256(N) (a skip layer's n + skip_n), pack_skip_tail_kernel writes the chunks past
// the last column tile in a second launch
int sr_tc_linear(const void* A, const void* W, const float* bias, int64_t M, int N, int K, int n_valid,
                 int act, int ch, void* A_next, int K_next, float scale, const float* skip_src,
                 int skip_n, int skip_ld, float* out, int out_ld, int out_col0, int out_n,
                 float* dstash, const void* mul_tiles, int mul_K, int mul_act, float mul_scale,
                 const int32_t* m_dev, cudaStream_t s) {
  using namespace sr_tc;
  if (M <= 0 || (ch != 1 && ch != 4)) return SR_EINVAL;
  if (!A || !W || !bias || N <= 0 || K <= 0 || (!A_next && !out)) return SR_EINVAL;
  if (mul_tiles ? (mul_K < n_valid || (mul_act != SR_ACT_NONE && mul_act != SR_ACT_SOFTPLUS100 && mul_act != SR_ACT_RELU))
                : (act < SR_ACT_NONE || act > SR_ACT_TANH))
    return SR_EINVAL;
  LayerArgs a;
  const int bn = tile_n(N);   // the column tile W was packed with (sr_tc_pack_weights of the same N)
  a.A = (const __nv_bfloat16*)A; a.W = (const __nv_bfloat16*)W; a.bias = bias; a.M = M;
  a.MT = (int)((M + BM - 1) / BM); a.NT = (N + bn - 1) / bn; a.KC = (K + 31) / 32;
  a.n_gemm = N; a.n = n_valid; a.ch = ch;
  a.A_next = (__nv_bfloat16*)A_next; a.KCn = A_next ? (K_next + 31) / 32 : 0;
  a.scale = scale; a.skip_src = skip_src; a.skip_n = skip_n; a.skip_ld = skip_ld;
  a.out = out; a.out_ld = out_ld; a.dstash = dstash; a.out_col0 = out_col0; a.out_n = out_n;
  a.mul_tiles = (const __nv_bfloat16*)mul_tiles; a.mul_KC = (mul_K + 31) / 32;
  a.mul_inv_scale = mul_scale != 0.f ? 1.0f / mul_scale : 1.0f; a.m_dev = m_dev;

  using Kern = void (*)(const LayerArgs);
  Kern kern = nullptr;
  const bool narrow = bn == BN_NARROW;
#define SR_SW(ACT_, CH_, MUL_)                                                                    \
  kern = narrow ? (Kern)tc_sweep_kernel<ACT_, CH_, MUL_, BN_NARROW> : (Kern)tc_sweep_kernel<ACT_, CH_, MUL_, BN>
  const int key = (ch == 4 ? 10 : 0) + (mul_tiles ? 5 + mul_act : act);
  switch (key) {
    case 0: SR_SW(SR_ACT_NONE, 1, false); break;
    case 1: SR_SW(SR_ACT_SOFTPLUS100, 1, false); break;
    case 2: SR_SW(SR_ACT_RELU, 1, false); break;
    case 3: SR_SW(SR_ACT_TANH, 1, false); break;
    case 5: SR_SW(SR_ACT_NONE, 1, true); break;
    case 6: SR_SW(SR_ACT_SOFTPLUS100, 1, true); break;
    case 7: SR_SW(SR_ACT_RELU, 1, true); break;
    case 10: SR_SW(SR_ACT_NONE, 4, false); break;
    case 11: SR_SW(SR_ACT_SOFTPLUS100, 4, false); break;
    case 12: SR_SW(SR_ACT_RELU, 4, false); break;
    case 13: SR_SW(SR_ACT_TANH, 4, false); break;
    case 15: SR_SW(SR_ACT_NONE, 4, true); break;
    case 16: SR_SW(SR_ACT_SOFTPLUS100, 4, true); break;
    case 17: SR_SW(SR_ACT_RELU, 4, true); break;
  }
#undef SR_SW
  if (!kern) return SR_EINVAL;
  // cudaFuncSetAttribute is per device: one flag per device ordinal (a process may drive several GPUs)
  static bool attr_set_dev[64][2][20] = {};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  bool& attr_set = attr_set_dev[cur_dev & 63][narrow][key];
  const size_t smem = narrow ? smem_bytes<BN_NARROW>() : smem_bytes<BN>();
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int grid = a.MT < SR_NUM_SMS ? a.MT : SR_NUM_SMS;
  kern<<<grid, kThreads, smem, s>>>(a);
  const int kc0 = a.NT * (bn / 32);   // first next-layer chunk the epilogue does not produce
  if (a.A_next != nullptr && a.KCn > kc0) {
    const int rc = sr_launch_status();
    if (rc) return rc;
    const long long total = (long long)a.MT * BM * (a.KCn - kc0) * 4;
    pack_skip_tail_kernel<<<sr_grid_for(total, 256, 8), 256, 0, s>>>(a.skip_src, a.skip_ld, a.n, a.skip_n, a.scale, M,
                                                                     kc0, a.KCn, a.A_next, m_dev);
  }
  return sr_launch_status();
}
}
