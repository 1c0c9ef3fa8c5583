// Fused MLP tile engine (device side) -- SURVEY.md rows a1-a4, a8.
//
// One CTA evaluates a whole MLP stack for a tile of kTileRows "rows" without leaving the SM:
// activations stay in shared memory (transposed, A_T[k][row]), the weights of each layer
// are streamed k-slice by k-slice from L2 into a shared-memory ring by the TMA engine
// (cp.async.bulk + mbarrier, issued by thread 0 one slice behind its own consumption), and 8
// warps run a register-tiled fp32 FFMA GEMM (8 rows x 16 cols per thread).
//
// Rows are (point, channel) pairs: channel 0 carries the value, channels 1..T carry
// forward-mode tangents d/dp_x, d/dp_y, d/dp_z, which share the layer GEMM with the value
// and are multiplied by act'(z_value) in the epilogue.  With T=3 one pass yields f and
// grad f (SDF) or the offset and its 3x3 Jacobian (deformer) -- no saved activations, no
// transposed weights, no second kernel.
//
// All arithmetic is fp32 (the ray finder's convergence test is |f| < 5e-5, SURVEY.md
// section 7 "hard parts"); this FFMA engine is the accuracy reference for the split-BF16
// tensor-core engine (tc_gemm.cu).
#pragma once
#include "common.cuh"

#ifndef SR_GEMM_UNROLL
#define SR_GEMM_UNROLL 8
#endif
#ifndef SR_WARPS
#define SR_WARPS 8        // 8: 8x16 thread tile, <=255 regs;  16: 8x8 thread tile, <=128 regs
#endif
#ifndef SR_FAST_ACT
#define SR_FAST_ACT 1     // MUFU-based softplus / sigmoid (abs. error < 3e-8 on activations)
#endif

namespace srmlp {

constexpr int kGemmUnroll = SR_GEMM_UNROLL;  // k-steps unrolled in the GEMM inner loop
constexpr int kTileRows = 64;          // rows per CTA tile
constexpr int kRowStride = 68;         // A_T row stride in floats (64 + 4 pad)
constexpr int kMaxK = 512;             // max fan-in (padded)
constexpr int kMaxN = 512;             // max fan-out (padded)
constexpr int kKT = 8;                 // k rows per pipeline stage
constexpr int kStages = 4;             // weight ring depth
constexpr int kStageFloats = kKT * kMaxN;
constexpr int kConsumerWarps = SR_WARPS;
constexpr int kConsumerThreads = kConsumerWarps * 32;
constexpr int kColSplit = kConsumerWarps / 8;      // warps sharing a row group split the column groups
constexpr int kAccCols = 16 / kColSplit;           // accumulator columns per thread
static_assert(kConsumerWarps == 8 || kConsumerWarps == 16, "8 or 16 warps");
// No dedicated producer warp: a 9th warp would put 3 warps on one SM sub-partition and cap
// every thread at 168 registers (spills in the 8x16 accumulator tile).  Thread 0 issues the
// TMA refills itself, one stage behind its own consumption (see Prod).
constexpr int kThreads = kConsumerThreads;
constexpr int kMaxIn = 296;            // max embedded input width kept in the stash (289 -> pad 8)
constexpr int kStashMax = 40;          // skip-connection stash: PE(3 + 6*6) = 39 -> 40

// Shared-memory carve-up (dynamic smem, 16-byte aligned pieces).
// One entry of the weight-streaming program of a tile: `nslices` bulk copies of `bytes` each.
struct Step {
  const char* src;
  uint32_t bytes;
  int nslices;
};
// The longest program is trace_rev_kernel's: forward and backward sweeps of the SDF and the translator, each up to
// SR_MLP_MAX_LAYERS steps.  program_add_* does not check the bound, so this must cover it.
constexpr int kMaxSteps = 4 * SR_MLP_MAX_LAYERS;

struct Smem {
  float* at;        // [kMaxK][kRowStride]
  float* wring;     // [kStages][kStageFloats]
  float* stash;     // [kStashMax][kRowStride]  embedded input kept for the skip layer
  float* res;       // [kTileRows][8] last-layer outputs (cols 0..7) per row
  uint64_t* full;   // [kStages]
  uint64_t* empty;  // [kStages]
  Step* steps;      // [kMaxSteps] weight-streaming program (same for every tile)
  int* nsteps;
};
constexpr size_t kSmemBytes = (size_t)kMaxK * kRowStride * 4 + (size_t)kStages * kStageFloats * 4 +
                              (size_t)kStashMax * kRowStride * 4 + (size_t)kTileRows * 8 * 4 +
                              2 * kStages * 8 + kMaxSteps * sizeof(Step) + 64;

__device__ __forceinline__ Smem carve(unsigned char* base) {
  Smem s;
  s.at = reinterpret_cast<float*>(base);
  base += (size_t)kMaxK * kRowStride * 4;
  s.wring = reinterpret_cast<float*>(base);
  base += (size_t)kStages * kStageFloats * 4;
  s.stash = reinterpret_cast<float*>(base);
  base += (size_t)kStashMax * kRowStride * 4;
  s.res = reinterpret_cast<float*>(base);
  base += (size_t)kTileRows * 8 * 4;
  s.full = reinterpret_cast<uint64_t*>(base);
  s.empty = s.full + kStages;
  base += 2 * kStages * 8;
  s.steps = reinterpret_cast<Step*>(base);
  base += kMaxSteps * sizeof(Step);
  s.nsteps = reinterpret_cast<int*>(base);
  return s;
}

// Ring position shared (by construction, not by memory) between producer and consumers:
// both walk exactly the same (tile, net, layer, k-slice) sequence.
struct Pipe {
  int slot;
  uint32_t phase;
  __device__ __forceinline__ void advance() {
    if (++slot == kStages) { slot = 0; phase ^= 1u; }
  }
};

__device__ __forceinline__ void pipe_init(const Smem& s) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      sr_mbar_init(&s.full[i], 1);
      sr_mbar_init(&s.empty[i], kConsumerWarps);
    }
    sr_fence_barrier_init();
  }
  __syncthreads();
}

// all-consumer barrier (named barrier 1; barrier 0 is left to __syncthreads)
__device__ __forceinline__ void consumer_sync() {
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
}

// ---------------------------------------------------------------------------------------------
// Weight-streaming program + producer cursor.
// The program (s.steps) lists, in consumption order, every GEMM of one tile: forward layers
// stream W_T k-slices, backward layers stream the un-transposed copy.  The cursor (meaningful
// in thread 0 only) walks tiles x steps x k-slices and issues one bulk copy per call: kStages-1
// slices up front, then one more each time warp 0 has finished a slice, so the slot it waits
// for is the one every warp finished a full slice ago (loose coupling, 3 slices in flight).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void program_begin(const Smem& s) {
  if (threadIdx.x == 0) *s.nsteps = 0;
}
__device__ __forceinline__ void program_add_fwd(const Smem& s, const sr_mlp_desc& net) {
  if (threadIdx.x == 0) {
    int n = *s.nsteps;
    for (int l = 0; l < net.n_layers; ++l, ++n) {
      const sr_mlp_layer& L = net.layer[l];
      s.steps[n].src = reinterpret_cast<const char*>(L.wt);
      s.steps[n].bytes = (uint32_t)(kKT * L.npad * 4);
      s.steps[n].nslices = L.kpad / kKT;
    }
    *s.nsteps = n;
  }
}
// backward GEMM of layer l: K = fan-out (padded to 8), N = fan-in (padded to 128)
__device__ __forceinline__ int bwd_kpad(const sr_mlp_layer& L) { return (L.n + kKT - 1) / kKT * kKT; }
__device__ __forceinline__ int bwd_npad(const sr_mlp_layer& L) { return (L.k + 127) / 128 * 128; }
__device__ __forceinline__ void program_add_bwd(const Smem& s, const sr_mlp_desc& net) {
  if (threadIdx.x == 0) {
    int n = *s.nsteps;
    for (int l = net.n_layers - 1; l >= 0; --l, ++n) {
      const sr_mlp_layer& L = net.layer[l];
      s.steps[n].src = reinterpret_cast<const char*>(L.wb);
      s.steps[n].bytes = (uint32_t)(kKT * bwd_npad(L) * 4);
      s.steps[n].nslices = bwd_kpad(L) / kKT;
    }
    *s.nsteps = n;
  }
}

struct Prod {
  Pipe pp;
  long long tile, ntiles;
  int stride, step, slice;
  bool done;
  __device__ __forceinline__ void init(long long first_tile, long long ntiles_, int stride_) {
    pp.slot = 0; pp.phase = 0;
    tile = first_tile; ntiles = ntiles_; stride = stride_;
    step = 0; slice = 0;
    done = first_tile >= ntiles_;
  }
  __device__ __forceinline__ void issue(const Smem& s) {
    if (done) return;
    const Step st = s.steps[step];
    sr_mbar_wait(&s.empty[pp.slot], pp.phase ^ 1u);
    sr_mbar_arrive_expect_tx(&s.full[pp.slot], st.bytes);
    sr_bulk_g2s(s.wring + (size_t)pp.slot * kStageFloats, st.src + (size_t)slice * st.bytes,
                st.bytes, &s.full[pp.slot]);
    pp.advance();
    if (++slice == st.nslices) {
      slice = 0;
      if (++step == *s.nsteps) {
        step = 0;
        tile += stride;
        if (tile >= ntiles) done = true;
      }
    }
  }
  // call after the program is complete; includes the barrier that publishes it
  __device__ __forceinline__ void prefill(const Smem& s) {
    __syncthreads();
    if (threadIdx.x == 0)
      for (int i = 0; i < kStages - 1; ++i) issue(s);
  }
};

// ---------------------------------------------------------------------------------------------
// Activations
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float softplus100(float z, float& deriv) {
  // torch.nn.Softplus(beta=100, threshold=20) and its autograd formula
  const float bz = z * 100.0f;
  if (bz > 20.0f) { deriv = 1.0f; return z; }
#if SR_FAST_ACT
  // MUFU.EX2 / MUFU.LG2 / fast divide: |error| <= ~3e-6 relative on e, i.e. < 3e-8 absolute on the
  // activation (values are O(0.01..1)); the libm path costs ~3x the instructions per element.
  const float e = __expf(bz);
  deriv = __fdividef(e, e + 1.0f);
  return __logf(1.0f + e) * 0.01f;
#else
  const float e = expf(bz);
  deriv = e / (e + 1.0f);
  return log1pf(e) / 100.0f;
#endif
}
// x / np.sqrt(2) of the skip connection (model/network.py:88-89)
__device__ __forceinline__ float div_sqrt2(float x) {
#if SR_FAST_ACT
  return x * 0.70710678118654752440f;
#else
  return __fdiv_rn(x, 1.41421356237309504880f);
#endif
}
__device__ __forceinline__ float apply_act(int act, float z, float& deriv) {
  switch (act) {
    case SR_ACT_SOFTPLUS100: return softplus100(z, deriv);
    case SR_ACT_RELU: deriv = z > 0.0f ? 1.0f : 0.0f; return z > 0.0f ? z : 0.0f;
    case SR_ACT_TANH: { const float t = tanhf(z); deriv = 1.0f - t * t; return t; }
    default: deriv = 1.0f; return z;
  }
}

// ---------------------------------------------------------------------------------------------
// One layer: acc = A_T[0:kpad][rows]^T * W_T[0:kpad][cols]
//   8 warps : thread (warp w, lane l) owns rows 8w..8w+7 and cols { g*128 + 4*l + i }, g < 4.
// ---------------------------------------------------------------------------------------------
// With 16 warps two warps share a row group and take alternate 128-column groups:
//   warp w: rows 8*(w%8).., groups { g*kColSplit + w/8 }.
template <int GP>
__device__ __forceinline__ void layer_gemm(const Smem& s, Pipe& cp, Prod& prod, int kpad,
                                           int npad, float (&acc)[8][kAccCols]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rg = warp & 7, ch = warp >> 3;
  const int ngroups = npad >> 7;
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int c = 0; c < kAccCols; ++c) acc[r][c] = 0.0f;
  const float* arow = s.at + 8 * rg;
  const int nslices = kpad / kKT;
  for (int sl = 0; sl < nslices; ++sl) {
    sr_mbar_wait(&s.full[cp.slot], cp.phase);
    const float* wst = s.wring + (size_t)cp.slot * kStageFloats + 4 * lane + ch * 128;
    const float* ak = arow + (size_t)sl * kKT * kRowStride;
#pragma unroll kGemmUnroll
    for (int kk = 0; kk < kKT; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(ak + kk * kRowStride);
      const float4 a1 = *reinterpret_cast<const float4*>(ak + kk * kRowStride + 4);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int g = 0; g < GP; ++g) {
        if (kColSplit == 1 || g * kColSplit + ch < ngroups) {
          const float4 w4 = *reinterpret_cast<const float4*>(wst + kk * npad + g * kColSplit * 128);
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            acc[r][4 * g + 0] = fmaf(a[r], w4.x, acc[r][4 * g + 0]);
            acc[r][4 * g + 1] = fmaf(a[r], w4.y, acc[r][4 * g + 1]);
            acc[r][4 * g + 2] = fmaf(a[r], w4.z, acc[r][4 * g + 2]);
            acc[r][4 * g + 3] = fmaf(a[r], w4.w, acc[r][4 * g + 3]);
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) sr_mbar_arrive(&s.empty[cp.slot]);
    if (threadIdx.x == 0) prod.issue(s);
    cp.advance();
  }
}

// Epilogue: bias + activation (+ tangent scaling), result back into A_T as the next layer's
// input, or -- for the last layer -- into s.res (cols < 8) and optionally a global feature
// buffer.  T = number of tangent channels (0 or 3): rows r of a thread are
//   T=0: 8 points;   T=3: 2 points x {value, d/dx, d/dy, d/dz}.
struct LastOut {
  float* feat;        // global [P][nfeat] or nullptr: cols 1..nfeat of value rows
  int nfeat;
  const int* row_pt;  // smem: global point index per tile-local point (or -1)
  float* dstash;      // global [n_layers][kMaxN][kTileRows] or nullptr: act'(z) of every hidden
                      // layer, kept for a reverse-mode pass over the same tile (T = 0 only)
};
constexpr size_t kDstashLayerFloats = (size_t)kMaxN * kTileRows;

template <int GP, int T>
__device__ __forceinline__ void layer_epilogue(const Smem& s, const sr_mlp_layer& L, int layer,
                                               bool last, bool next_skip, int next_kpad, int d_in,
                                               const LastOut& lo, float (&acc)[8][kAccCols]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rg = warp & 7, ch = warp >> 3;
  constexpr int CH = T + 1;
  constexpr int PPT = 8 / CH;  // points per thread
  // (1) every warp must be done reading A_T before anyone overwrites it
  consumer_sync();
#pragma unroll
  for (int g = 0; g < GP; ++g) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = 4 * g + i;
      const int col = (g * kColSplit + ch) * 128 + 4 * lane + i;
      if (col < L.n) {
        const float b = __ldg(L.bias + col);
        float o[8];
        float dv[8];
#pragma unroll
        for (int p = 0; p < PPT; ++p) {
          float d;
          const float z = acc[p * CH][c] + b;
          o[p * CH] = apply_act(L.act, z, d);
          dv[p] = d;
#pragma unroll
          for (int t = 1; t < CH; ++t) o[p * CH + t] = d * acc[p * CH + t][c];
        }
        if (T == 0 && !last && lo.dstash != nullptr) {
          float* dd = lo.dstash + (size_t)layer * kDstashLayerFloats + (size_t)col * kTileRows + 8 * rg;
          *reinterpret_cast<float4*>(dd) = make_float4(dv[0], dv[1], dv[2], dv[3]);
          *reinterpret_cast<float4*>(dd + 4) = make_float4(dv[4], dv[5], dv[6], dv[7]);
        }
        if (!last) {
          if (next_skip) {
#pragma unroll
            for (int r = 0; r < 8; ++r) o[r] = div_sqrt2(o[r]);
          }
          float* dst = s.at + (size_t)col * kRowStride + 8 * rg;
          *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
          *reinterpret_cast<float4*>(dst + 4) = make_float4(o[4], o[5], o[6], o[7]);
        } else {
          if (col < 8) {
#pragma unroll
            for (int r = 0; r < 8; ++r) s.res[(8 * rg + r) * 8 + col] = o[r];
          }
          if (lo.feat != nullptr && col >= 1 && col <= lo.nfeat) {
#pragma unroll
            for (int p = 0; p < PPT; ++p) {
              const int gp = lo.row_pt[(8 * rg) / CH + p];
              if (gp >= 0) lo.feat[(size_t)gp * lo.nfeat + (col - 1)] = o[p * CH];
            }
          }
        }
      } else if (!last) {
        // zero the k-padding rows the next layer will multiply by zero weights
        const int lim = next_skip ? 0 : next_kpad;  // (skip case handled below)
        if (col < lim) {
          float* dst = s.at + (size_t)col * kRowStride + 8 * rg;
          *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
          *reinterpret_cast<float4*>(dst + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
  }
  if (!last && next_skip) {
    // x = cat([x, input]) / sqrt(2): append the stashed embedded input (model/network.py:88-89)
    for (int idx = threadIdx.x; idx < (next_kpad - L.n) * (kTileRows / 4); idx += kConsumerThreads) {
      const int kk = idx / (kTileRows / 4), r4 = (idx % (kTileRows / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kk < d_in) {
        v = *reinterpret_cast<const float4*>(s.stash + (size_t)kk * kRowStride + r4);
        v.x = div_sqrt2(v.x); v.y = div_sqrt2(v.y); v.z = div_sqrt2(v.z); v.w = div_sqrt2(v.w);
      }
      *reinterpret_cast<float4*>(s.at + (size_t)(L.n + kk) * kRowStride + r4) = v;
    }
  }
  // (2) next layer's reads must see the writes
  consumer_sync();
}

// Runs all layers of `net` on the tile whose embedded input is already in A_T rows
// [0, layer[0].kpad) (and in the stash when the net has a skip layer).
template <int T>
__device__ __forceinline__ void run_net(const sr_mlp_desc& net, const Smem& s, Pipe& cp,
                                        Prod& prod, const LastOut& lo) {
  float acc[8][kAccCols];
  for (int l = 0; l < net.n_layers; ++l) {
    const sr_mlp_layer& L = net.layer[l];
    const bool last = (l == net.n_layers - 1);
    const bool next_skip = !last && net.layer[l + 1].skip != 0;
    const int next_kpad = last ? 0 : net.layer[l + 1].kpad;
    const int gp = ((L.npad >> 7) + kColSplit - 1) / kColSplit;  // column groups per thread
    if (kColSplit == 2) {
      if (gp == 1) {
        layer_gemm<1>(s, cp, prod, L.kpad, L.npad, acc);
        layer_epilogue<1, T>(s, L, l, last, next_skip, next_kpad, net.d_in, lo, acc);
      } else {
        layer_gemm<(kColSplit == 2 ? 2 : 1)>(s, cp, prod, L.kpad, L.npad, acc);
        layer_epilogue<(kColSplit == 2 ? 2 : 1), T>(s, L, l, last, next_skip, next_kpad, net.d_in, lo, acc);
      }
    } else {
      switch (gp) {
        case 1:
          layer_gemm<1>(s, cp, prod, L.kpad, L.npad, acc);
          layer_epilogue<1, T>(s, L, l, last, next_skip, next_kpad, net.d_in, lo, acc);
          break;
        case 2:
          layer_gemm<(kColSplit == 1 ? 2 : 1)>(s, cp, prod, L.kpad, L.npad, acc);
          layer_epilogue<(kColSplit == 1 ? 2 : 1), T>(s, L, l, last, next_skip, next_kpad, net.d_in, lo, acc);
          break;
        case 3:
          layer_gemm<(kColSplit == 1 ? 3 : 1)>(s, cp, prod, L.kpad, L.npad, acc);
          layer_epilogue<(kColSplit == 1 ? 3 : 1), T>(s, L, l, last, next_skip, next_kpad, net.d_in, lo, acc);
          break;
        default:
          layer_gemm<(kColSplit == 1 ? 4 : 1)>(s, cp, prod, L.kpad, L.npad, acc);
          layer_epilogue<(kColSplit == 1 ? 4 : 1), T>(s, L, l, last, next_skip, next_kpad, net.d_in, lo, acc);
          break;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Reverse-mode pass over the tile that run_net<0> just evaluated with a derivative stash.
//   in : A_T rows [0, bwd_kpad(last)) hold the cotangent of the net's outputs (row k = output k)
//   out: A_T rows [0, d_in) hold d(sum_k cot_k * out_k) / d(embedded input)   (skip path included)
// Backward GEMM of layer l: g_in[rows x fan_in] = delta_l[rows x fan_out] * W_l, streamed from the
// un-transposed padded copy `wb`; delta_{l-1} = g_in * act'_{l-1} (and the /sqrt(2) of a skip).
// ---------------------------------------------------------------------------------------------
template <int GP>
__device__ __forceinline__ void bwd_epilogue(const Smem& s, const sr_mlp_desc& net, int l,
                                             const float* dstash, float (&acc)[8][kAccCols]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rg = warp & 7, ch = warp >> 3;
  const sr_mlp_layer& L = net.layer[l];
  const bool skip = L.skip != 0;
  const int n_prev = l > 0 ? net.layer[l - 1].n : 0;         // width of the previous layer's output
  const int next_k = l > 0 ? bwd_kpad(net.layer[l - 1]) : 0;  // K of the next backward GEMM
  consumer_sync();
  const int ngroups = bwd_npad(L) >> 7;
#pragma unroll
  for (int g = 0; g < GP; ++g) {
    if (kColSplit == 2 && g * kColSplit + ch >= ngroups) continue;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = 4 * g + i;
      const int col = (g * kColSplit + ch) * 128 + 4 * lane + i;
      float o[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) o[r] = acc[r][c];
      if (skip) {
#pragma unroll
        for (int r = 0; r < 8; ++r) o[r] = div_sqrt2(o[r]);
      }
      if (l == 0) {
        if (col < L.k) {
          float* dst = s.at + (size_t)col * kRowStride + 8 * rg;
          if (col < kStashMax) {  // add the gradient that arrived through the skip connection
            const float* sg = s.stash + (size_t)col * kRowStride + 8 * rg;
#pragma unroll
            for (int r = 0; r < 8; ++r) o[r] += sg[r];
          }
          *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
          *reinterpret_cast<float4*>(dst + 4) = make_float4(o[4], o[5], o[6], o[7]);
        }
      } else if (col < n_prev) {
        const float* dd = dstash + (size_t)(l - 1) * kDstashLayerFloats + (size_t)col * kTileRows + 8 * rg;
        const float4 d0 = *reinterpret_cast<const float4*>(dd);
        const float4 d1 = *reinterpret_cast<const float4*>(dd + 4);
        float* dst = s.at + (size_t)col * kRowStride + 8 * rg;
        *reinterpret_cast<float4*>(dst) = make_float4(o[0] * d0.x, o[1] * d0.y, o[2] * d0.z, o[3] * d0.w);
        *reinterpret_cast<float4*>(dst + 4) = make_float4(o[4] * d1.x, o[5] * d1.y, o[6] * d1.z, o[7] * d1.w);
      } else {
        if (skip && col < n_prev + net.d_in && col - n_prev < kStashMax) {
          // accumulate: every skip layer adds its share of the embedded input's gradient
          float* sg = s.stash + (size_t)(col - n_prev) * kRowStride + 8 * rg;
          const float4 s0 = *reinterpret_cast<const float4*>(sg);
          const float4 s1 = *reinterpret_cast<const float4*>(sg + 4);
          *reinterpret_cast<float4*>(sg) = make_float4(s0.x + o[0], s0.y + o[1], s0.z + o[2], s0.w + o[3]);
          *reinterpret_cast<float4*>(sg + 4) = make_float4(s1.x + o[4], s1.y + o[5], s1.z + o[6], s1.w + o[7]);
        }
        if (col < next_k) {  // k-padding of the next backward GEMM
          float* dst = s.at + (size_t)col * kRowStride + 8 * rg;
          *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
          *reinterpret_cast<float4*>(dst + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
  }
  consumer_sync();
}

// zero the skip-gradient stash (call before run_net_bwd on a net; cheap: 40 x 64 floats)
__device__ __forceinline__ void bwd_clear_stash(const Smem& s) {
  for (int idx = threadIdx.x; idx < kStashMax * (kTileRows / 4); idx += kConsumerThreads) {
    const int k = idx / (kTileRows / 4), r4 = (idx % (kTileRows / 4)) * 4;
    *reinterpret_cast<float4*>(s.stash + (size_t)k * kRowStride + r4) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__device__ __forceinline__ void run_net_bwd(const sr_mlp_desc& net, const Smem& s, Pipe& cp,
                                            Prod& prod, const float* dstash) {
  float acc[8][kAccCols];
  for (int l = net.n_layers - 1; l >= 0; --l) {
    const sr_mlp_layer& L = net.layer[l];
    const int kp = bwd_kpad(L), np = bwd_npad(L);
    const int gp = ((np >> 7) + kColSplit - 1) / kColSplit;
    if (kColSplit == 2) {
      if (gp == 1) { layer_gemm<1>(s, cp, prod, kp, np, acc); bwd_epilogue<1>(s, net, l, dstash, acc); }
      else { layer_gemm<(kColSplit == 2 ? 2 : 1)>(s, cp, prod, kp, np, acc); bwd_epilogue<(kColSplit == 2 ? 2 : 1)>(s, net, l, dstash, acc); }
    } else {
      switch (gp) {
        case 1: layer_gemm<1>(s, cp, prod, kp, np, acc); bwd_epilogue<1>(s, net, l, dstash, acc); break;
        case 2: layer_gemm<(kColSplit == 1 ? 2 : 1)>(s, cp, prod, kp, np, acc); bwd_epilogue<(kColSplit == 1 ? 2 : 1)>(s, net, l, dstash, acc); break;
        case 3: layer_gemm<(kColSplit == 1 ? 3 : 1)>(s, cp, prod, kp, np, acc); bwd_epilogue<(kColSplit == 1 ? 3 : 1)>(s, net, l, dstash, acc); break;
        default: layer_gemm<(kColSplit == 1 ? 4 : 1)>(s, cp, prod, kp, np, acc); bwd_epilogue<(kColSplit == 1 ? 4 : 1)>(s, net, l, dstash, acc); break;
      }
    }
  }
}

// chain rule through the positional encoding: rows [0, 3+6L) of A_T hold dL/d(embedding);
// returns dL/dx for tile row `row` at point x.
__device__ __forceinline__ void embed_backward(const float* at, int row, const float x[3],
                                               int multires, const float* pe_w, float g[3]) {
#pragma unroll
  for (int j = 0; j < 3; ++j) g[j] = at[(size_t)j * kRowStride + row];
  float freq = 1.0f;
  for (int b = 0; b < multires; ++b, freq *= 2.0f) {
    const float w = pe_w[b] * freq;
    const int ks = 3 + 6 * b, kc = ks + 3;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float sn, cs;
      sincosf(x[j] * freq, &sn, &cs);
      g[j] += w * (cs * at[(size_t)(ks + j) * kRowStride + row] - sn * at[(size_t)(kc + j) * kRowStride + row]);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Positional encoding of a 3-vector into A_T rows [k0, k0 + 3 + 6*L) for tile row `row`
// (value channel) and, if T=3, its three tangent rows (row+1..row+3).
//   layout (model/Embedder.py:11-32): [x, sin(2^0 x), cos(2^0 x), sin(2^1 x), cos(2^1 x), ...]
//   each block 3 wide; band weights w_b (utils/utils.py:40-46) multiply sin and cos.
// ---------------------------------------------------------------------------------------------
template <int T>
__device__ __forceinline__ void embed_point(float* dst, int k0, int row, const float x[3],
                                            int multires, const float* pe_w, bool tangent_unit) {
  // value row
#pragma unroll
  for (int j = 0; j < 3; ++j) dst[(size_t)(k0 + j) * kRowStride + row] = x[j];
  if (T == 3) {
#pragma unroll
    for (int t = 0; t < 3; ++t)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        dst[(size_t)(k0 + j) * kRowStride + row + 1 + t] = (tangent_unit && t == j) ? 1.0f : 0.0f;
  }
  float freq = 1.0f;
  for (int b = 0; b < multires; ++b, freq *= 2.0f) {
    const float w = pe_w[b];
    const int ks = k0 + 3 + 6 * b, kc = ks + 3;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const float arg = x[j] * freq;
      float sn, cs;
      sincosf(arg, &sn, &cs);
      dst[(size_t)(ks + j) * kRowStride + row] = w * sn;
      dst[(size_t)(kc + j) * kRowStride + row] = w * cs;
      if (T == 3) {
#pragma unroll
        for (int t = 0; t < 3; ++t) {
          const bool on = tangent_unit && (t == j);
          dst[(size_t)(ks + j) * kRowStride + row + 1 + t] = on ? (w * freq) * cs : 0.0f;
          dst[(size_t)(kc + j) * kRowStride + row + 1 + t] = on ? -(w * freq) * sn : 0.0f;
        }
      }
    }
  }
}

}  // namespace srmlp
