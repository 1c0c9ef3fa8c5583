// Fused field kernels built on the tile engine in mlp_core.cuh:
//   sdf_kernel      ImplicitNetwork.forward / .gradient          (model/network.py:72-114)
//   deform_kernel   CompositeDeformer = MLPTranslator + LBSkinner (model/Deformer.py:10-233)
//   render_kernel   RenderingNetwork_view_norm.forward            (model/RenderNet.py:54-89)
//   trace_kernel    one iteration of OptimizeSurfacePs            (utils/FindSurfacePs.py:114-163)
//   shade_kernel    normals + cardinal rays + features            (utils/utils.py:132-169)
//   fold / bone-transform / re-layout helpers.
// Every kernel is persistent (grid = #SMs, tiles strided across CTAs), 8 warps, thread 0
// doubling as the TMA producer, ~221 KB dynamic shared memory, one CTA per SM.
#include "mlp_core.cuh"
#include "lbs.cuh"
#include "trace_rules.cuh"

using namespace srmlp;

namespace {

// aux per tile-local point (floats / int bit patterns)
constexpr int kAuxStride = 32;
enum {
  AUX_P = 0,      // 3: canonical point
  AUX_GP = 3,     // global point index (int), -1 = padding
  AUX_B = 4,      // frame / batch index (int)
  AUX_F = 5,      // sdf value
  AUX_GF = 6,     // 3: grad f
  AUX_D = 9,      // 3: deformed point
  AUX_J = 12,     // 9: Jacobian dD/dp
  AUX_OFF = 21,   // 3: translator offset
  AUX_CI = 24,    // 3: lbs corner indices (int)
};
constexpr size_t kAuxBytes = (size_t)kTileRows * kAuxStride * 4;
constexpr size_t kDynSmem = kSmemBytes + kAuxBytes + 256 /*row_pt*/ + 128 /*align*/;
static_assert(kDynSmem <= 232448, "exceeds the H100's 227 KB of dynamic shared memory per block");

struct TileCtx {
  Smem s;
  float* aux;   // [kTileRows][kAuxStride]
  int* row_pt;  // [kTileRows] global point per local point
};

__device__ __forceinline__ TileCtx make_ctx(unsigned char* raw) {
  // `raw` is the __align__(128) dynamic shared array itself: no integer round trip, so the
  // compiler keeps the shared address space and emits LDS/STS instead of generic LD/ST.
  unsigned char* base = raw;
  TileCtx c;
  c.s = carve(base);
  base += (kSmemBytes + 15) & ~size_t(15);
  c.aux = reinterpret_cast<float*>(base);
  base += kAuxBytes;
  c.row_pt = reinterpret_cast<int*>(base);
  return c;
}

// ---------------------------------------------------------------------------------------------
// Tile setup: which global points does this tile hold?
// ---------------------------------------------------------------------------------------------
template <int T>
__device__ __forceinline__ void load_points(const TileCtx& c, long long tile, long long count,
                                            const int32_t* __restrict__ index,
                                            const float* __restrict__ pts,
                                            const int64_t* __restrict__ batch_inds,
                                            long long pts_per_frame) {
  constexpr int PTS = kTileRows / (T + 1);
  const int pl = threadIdx.x;
  if (pl < PTS) {
    const long long li = tile * PTS + pl;
    float* a = c.aux + pl * kAuxStride;
    int gp = -1, b = 0;
    float x = 0.f, y = 0.f, z = 0.f;
    if (li < count) {
      gp = index ? index[li] : (int)li;
      x = pts[(size_t)gp * 3 + 0];
      y = pts[(size_t)gp * 3 + 1];
      z = pts[(size_t)gp * 3 + 2];
      if (batch_inds) b = (int)batch_inds[gp];
      else if (pts_per_frame > 0) b = (int)(gp / pts_per_frame);
    }
    a[AUX_P + 0] = x; a[AUX_P + 1] = y; a[AUX_P + 2] = z;
    a[AUX_GP] = __int_as_float(gp);
    a[AUX_B] = __int_as_float(b);
    c.row_pt[pl] = gp;
  }
}

// Embedded input of the SDF / translator nets: PE(p) [+ cond[b]] into A_T, zero k-padding,
// copy to the skip stash when the net has a skip layer.
template <int T>
__device__ __forceinline__ void prologue_pe(const TileCtx& c, const sr_mlp_desc& net,
                                            const float* __restrict__ conds, int condlen) {
  constexpr int CH = T + 1, PTS = kTileRows / CH;
  const int pe_dim = 3 + 6 * net.multires;
  if (threadIdx.x < PTS) {
    const float* a = c.aux + threadIdx.x * kAuxStride;
    const float x[3] = {a[AUX_P], a[AUX_P + 1], a[AUX_P + 2]};
    const bool valid = __float_as_int(a[AUX_GP]) >= 0;
    embed_point<T>(c.s.at, 0, threadIdx.x * CH, x, net.multires, net.pe_w, valid);
  }
  const int kpad0 = net.layer[0].kpad;
  // conditioning vector (value rows only; it does not depend on p) + zero padding
  for (int idx = threadIdx.x; idx < (kpad0 - pe_dim) * kTileRows; idx += kConsumerThreads) {
    const int k = pe_dim + idx / kTileRows, row = idx % kTileRows;
    float v = 0.0f;
    const int kc = k - pe_dim;
    if (kc < condlen && (row % CH) == 0) {
      const float* a = c.aux + (row / CH) * kAuxStride;
      if (__float_as_int(a[AUX_GP]) >= 0)
        v = __ldg(conds + (size_t)__float_as_int(a[AUX_B]) * condlen + kc);
    }
    c.s.at[(size_t)k * kRowStride + row] = v;
  }
  consumer_sync();
  bool has_skip = false;
  for (int l = 0; l < net.n_layers; ++l) has_skip |= net.layer[l].skip != 0;
  if (has_skip) {
    for (int idx = threadIdx.x; idx < net.d_in * (kTileRows / 4); idx += kConsumerThreads) {
      const int k = idx / (kTileRows / 4), r4 = (idx % (kTileRows / 4)) * 4;
      *reinterpret_cast<float4*>(c.s.stash + (size_t)k * kRowStride + r4) =
          *reinterpret_cast<const float4*>(c.s.at + (size_t)k * kRowStride + r4);
    }
    // (visibility is guaranteed by the barriers inside the first layer's epilogue)
  }
}

// After run_net<T>(translator): res holds offset (+ tangents).  Computes D(p) and, for T=3,
// J = dD/dp into aux.  One warp per point.
template <int T>
__device__ __forceinline__ void deform_finish(const TileCtx& c, const sr_lbs_params* lbs) {
  constexpr int CH = T + 1, PTS = kTileRows / CH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int pl = warp; pl < PTS; pl += kConsumerWarps) {
    float* a = c.aux + pl * kAuxStride;
    const int row = pl * CH;
    float off[3], pp[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      off[j] = c.s.res[row * 8 + j];
      pp[j] = __fadd_rn(a[AUX_P + j], off[j]);
    }
    float d[3], M[9];
    int ci[3] = {0, 0, 0};
    if (lbs) {
      lbs_point(*lbs, pp, __float_as_int(a[AUX_B]), d, M, ci);
    } else {
#pragma unroll
      for (int j = 0; j < 3; ++j) d[j] = pp[j];
#pragma unroll
      for (int i = 0; i < 9; ++i) M[i] = (i % 4 == 0) ? 1.f : 0.f;
    }
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        a[AUX_D + j] = d[j];
        a[AUX_OFF + j] = off[j];
        a[AUX_CI + j] = __int_as_float(ci[j]);
      }
      if (T == 0) {
        // reverse-mode callers need M = dD/dp' (the translator Jacobian comes from the backward sweep)
#pragma unroll
        for (int i = 0; i < 9; ++i) a[AUX_J + i] = M[i];
      }
      if (T == 3) {
        // dp'/dp = I + Joff, Joff[m][cc] = d off_m / d p_cc = res[row+1+cc][m]
        float Q[9];
#pragma unroll
        for (int m = 0; m < 3; ++m)
#pragma unroll
          for (int cc = 0; cc < 3; ++cc)
            Q[3 * m + cc] = (m == cc ? 1.f : 0.f) + c.s.res[(row + 1 + cc) * 8 + m];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int cc = 0; cc < 3; ++cc)
            a[AUX_J + 3 * r + cc] =
                M[3 * r] * Q[cc] + M[3 * r + 1] * Q[3 + cc] + M[3 * r + 2] * Q[6 + cc];
      }
    }
  }
}

// SDF results (res) -> aux
template <int T>
__device__ __forceinline__ void sdf_finish(const TileCtx& c) {
  constexpr int CH = T + 1, PTS = kTileRows / CH;
  if (threadIdx.x < PTS) {
    float* a = c.aux + threadIdx.x * kAuxStride;
    const int row = threadIdx.x * CH;
    a[AUX_F] = c.s.res[row * 8];
    if (T == 3) {
#pragma unroll
      for (int t = 0; t < 3; ++t) a[AUX_GF + t] = c.s.res[(row + 1 + t) * 8];
    }
  }
}

// identity deformer: D(p) = p, J = I
template <int T>
__device__ __forceinline__ void identity_deform(const TileCtx& c) {
  constexpr int PTS = kTileRows / (T + 1);
  if (threadIdx.x < PTS) {
    float* a = c.aux + threadIdx.x * kAuxStride;
#pragma unroll
    for (int j = 0; j < 3; ++j) { a[AUX_D + j] = a[AUX_P + j]; a[AUX_OFF + j] = 0.f; }
#pragma unroll
    for (int i = 0; i < 9; ++i) a[AUX_J + i] = (i % 4 == 0) ? 1.f : 0.f;
  }
}

// =============================================================================================
// Kernels
// =============================================================================================
struct SdfArgs {
  sr_mlp_desc net;
  const float* pts;
  long long P;
  float* sdf;
  float* grad;
  float* feat;
  int nfeat;
  const int32_t* index;   // optional list of point ids to evaluate (results land at sdf[id])
  const int32_t* m_dev;   // device-side length of `index`
};

template <int T>
__global__ void __launch_bounds__(kThreads, 1) sdf_kernel(const __grid_constant__ SdfArgs args) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileCtx c = make_ctx(smem_raw);
  pipe_init(c.s);
  constexpr int PTS = kTileRows / (T + 1);
  long long count = args.P;
  if (args.m_dev != nullptr) { const long long md = *args.m_dev; count = md < count ? md : count; }
  const long long ntiles = (count + PTS - 1) / PTS;
  Pipe cp{0, 0};
  Prod prod;
  program_begin(c.s);
  program_add_fwd(c.s, args.net);
  prod.init(blockIdx.x, ntiles, gridDim.x);
  prod.prefill(c.s);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    load_points<T>(c, tile, count, args.index, args.pts, nullptr, 0);
    consumer_sync();
    prologue_pe<T>(c, args.net, nullptr, 0);
    LastOut lo{args.feat, args.nfeat, c.row_pt, nullptr};
    run_net<T>(args.net, c.s, cp, prod, lo);
    if (threadIdx.x < PTS) {
      const int gp = c.row_pt[threadIdx.x];
      if (gp >= 0) {
        const int row = threadIdx.x * (T + 1);
        args.sdf[gp] = c.s.res[row * 8];
        if (T == 3) {
#pragma unroll
          for (int t = 0; t < 3; ++t) args.grad[(size_t)gp * 3 + t] = c.s.res[(row + 1 + t) * 8];
        }
      }
    }
    consumer_sync();
  }
}

struct DeformArgs {
  sr_mlp_desc net;
  sr_lbs_params lbs;
  int has_lbs;
  const float* pts;
  const int64_t* batch_inds;
  long long pts_per_frame;
  const float* conds;
  int condlen;
  long long P;
  float* d;
  float* offset;
  float* jac;
  int32_t* corner_idx;
};

template <int T>
__global__ void __launch_bounds__(kThreads, 1)
deform_kernel(const __grid_constant__ DeformArgs args) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileCtx c = make_ctx(smem_raw);
  pipe_init(c.s);
  constexpr int PTS = kTileRows / (T + 1);
  const long long ntiles = (args.P + PTS - 1) / PTS;
  Pipe cp{0, 0};
  Prod prod;
  program_begin(c.s);
  program_add_fwd(c.s, args.net);
  prod.init(blockIdx.x, ntiles, gridDim.x);
  prod.prefill(c.s);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    load_points<T>(c, tile, args.P, nullptr, args.pts, args.batch_inds, args.pts_per_frame);
    consumer_sync();
    prologue_pe<T>(c, args.net, args.conds, args.condlen);
    LastOut lo{nullptr, 0, c.row_pt, nullptr};
    run_net<T>(args.net, c.s, cp, prod, lo);
    deform_finish<T>(c, args.has_lbs ? &args.lbs : nullptr);
    consumer_sync();
    if (threadIdx.x < PTS) {
      const float* a = c.aux + threadIdx.x * kAuxStride;
      const int gp = __float_as_int(a[AUX_GP]);
      if (gp >= 0) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          args.d[(size_t)gp * 3 + j] = a[AUX_D + j];
          if (args.offset) args.offset[(size_t)gp * 3 + j] = a[AUX_OFF + j];
          if (args.corner_idx) args.corner_idx[(size_t)gp * 3 + j] = __float_as_int(a[AUX_CI + j]);
        }
        if (T == 3 && args.jac) {
#pragma unroll
          for (int i = 0; i < 9; ++i) args.jac[(size_t)gp * 9 + i] = a[AUX_J + i];
        }
      }
    }
    consumer_sync();
  }
}

struct RenderArgs {
  sr_mlp_desc net;
  const float* pts;
  const float* normals;
  const float* views;
  const float* feat;
  int nfeat;
  long long P;
  float* rgb;
};

__global__ void __launch_bounds__(kThreads, 1)
render_kernel(const __grid_constant__ RenderArgs args) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileCtx c = make_ctx(smem_raw);
  pipe_init(c.s);
  const long long ntiles = (args.P + kTileRows - 1) / kTileRows;
  Pipe cp{0, 0};
  Prod prod;
  program_begin(c.s);
  program_add_fwd(c.s, args.net);
  prod.init(blockIdx.x, ntiles, gridDim.x);
  prod.prefill(c.s);
  const sr_mlp_desc& net = args.net;
  const int pe_dim = 3 + 6 * net.multires;  // embedded view direction
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    // rendering_input = cat([points, PE(view_dirs), normals, feature_vectors])
    if (threadIdx.x < kTileRows) {
      const long long gp = tile * kTileRows + threadIdx.x;
      const bool valid = gp < args.P;
      c.row_pt[threadIdx.x] = valid ? (int)gp : -1;
      float p[3] = {0.f, 0.f, 0.f}, v[3] = {0.f, 0.f, 0.f}, n[3] = {0.f, 0.f, 0.f};
      if (valid) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          p[j] = args.pts[gp * 3 + j];
          v[j] = args.views[gp * 3 + j];
          n[j] = args.normals[gp * 3 + j];
        }
      }
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        c.s.at[(size_t)j * kRowStride + threadIdx.x] = p[j];
        c.s.at[(size_t)(3 + pe_dim + j) * kRowStride + threadIdx.x] = n[j];
      }
      embed_point<0>(c.s.at, 3, threadIdx.x, v, net.multires, net.pe_w, false);
    }
    const int k0 = 3 + pe_dim + 3;
    const int kpad0 = net.layer[0].kpad;
    // features: coalesced over k for each row
    for (int idx = threadIdx.x; idx < (kpad0 - k0) * kTileRows; idx += kConsumerThreads) {
      const int row = idx / (kpad0 - k0), kf = idx % (kpad0 - k0);
      const long long gp = tile * kTileRows + row;
      float v = 0.f;
      if (gp < args.P && kf < args.nfeat) v = __ldg(args.feat + (size_t)gp * args.nfeat + kf);
      c.s.at[(size_t)(k0 + kf) * kRowStride + row] = v;
    }
    consumer_sync();
    LastOut lo{nullptr, 0, c.row_pt, nullptr};
    run_net<0>(net, c.s, cp, prod, lo);
    if (threadIdx.x < kTileRows) {
      const int gp = c.row_pt[threadIdx.x];
      if (gp >= 0) {
#pragma unroll
        for (int j = 0; j < 3; ++j) args.rgb[(size_t)gp * 3 + j] = c.s.res[threadIdx.x * 8 + j];
      }
    }
    consumer_sync();
  }
}

// ---------------------------------------------------------------------------------------------
// Surface-point finder: one launch = evaluate f, grad f, D, J at the current points of the
// active list, test convergence, take one damped Newton step on the unconverged ones.
// ---------------------------------------------------------------------------------------------
struct TraceArgs {
  sr_mlp_desc sdf;
  sr_mlp_desc dnet;
  sr_lbs_params lbs;
  int has_lbs;
  int has_dnet;  // 0: identity deformer D(p) = p (BASELINE config 1)
  sr_trace_params tp;
  float* pts;
  const float* rays;
  const int64_t* batch_inds;
  const float* conds;
  int condlen;
  long long P;
  const int32_t* active_in;  // nullptr: identity list of length P (first launch)
  int32_t* active_out;
  int32_t* counters;         // counters[iter] = |active_in|, counters[iter+1] += survivors
  int iter;
  int do_update;             // 0 on the final (test-only) launch
  uint8_t* converged;
};

__global__ void __launch_bounds__(kThreads, 1)
trace_kernel(const __grid_constant__ TraceArgs args) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileCtx c = make_ctx(smem_raw);
  pipe_init(c.s);
  constexpr int T = 3, PTS = kTileRows / (T + 1);
  const long long count = args.active_in ? (long long)args.counters[args.iter] : args.P;
  const long long ntiles = (count + PTS - 1) / PTS;
  Pipe cp{0, 0};
  Prod prod;
  program_begin(c.s);
  program_add_fwd(c.s, args.sdf);
  if (args.has_dnet) program_add_fwd(c.s, args.dnet);
  prod.init(blockIdx.x, ntiles, gridDim.x);
  prod.prefill(c.s);
  const LastOut lo{nullptr, 0, c.row_pt, nullptr};
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    load_points<T>(c, tile, count, args.active_in, args.pts, args.batch_inds, 0);
    consumer_sync();
    prologue_pe<T>(c, args.sdf, nullptr, 0);
    run_net<T>(args.sdf, c.s, cp, prod, lo);
    sdf_finish<T>(c);
    consumer_sync();
    if (args.has_dnet) {
      prologue_pe<T>(c, args.dnet, args.conds, args.condlen);
      run_net<T>(args.dnet, c.s, cp, prod, lo);
      deform_finish<T>(c, args.has_lbs ? &args.lbs : nullptr);
    } else {
      identity_deform<T>(c);
    }
    consumer_sync();
    if (threadIdx.x < PTS) {
      const float* a = c.aux + threadIdx.x * kAuxStride;
      const int gp = __float_as_int(a[AUX_GP]);
      if (gp >= 0) {
        const float f = a[AUX_F];
        const RayTest r = ray_test(f, a + AUX_D, args.rays + (size_t)gp * 3, args.tp);
        if (r.done) {
          args.converged[gp] = 1;
        } else if (args.do_update) {
          // g = d loss / d p = w1 sign(f) grad f + w2 J^T q
          float u[3];
          const float loss = ray_loss(r, f, a + AUX_J, args.tp, u);
          const float cot_f = sdf_cotangent(f, args.tp);
          float g[3];
#pragma unroll
          for (int j = 0; j < 3; ++j) g[j] = cot_f * a[AUX_GF + j] + u[j];
          newton_step(args.pts + (size_t)gp * 3, a + AUX_P, g, loss, &args.counters[args.iter + 1], args.active_out,
                      gp);
        }
      }
    }
    consumer_sync();
  }
}

// ---------------------------------------------------------------------------------------------
// Reverse-mode tracer step: 64 rays per tile, value-only forward sweeps that stash act'(z),
// then one backward sweep per network with the loss cotangent.  Same update as trace_kernel.
// ---------------------------------------------------------------------------------------------
struct TraceRevArgs {
  TraceArgs t;
  float* scratch;  // [gridDim.x][2][SR_MLP_MAX_LAYERS][kMaxN][kTileRows]
};
constexpr size_t kScratchPerCta = 2 * (size_t)SR_MLP_MAX_LAYERS * kDstashLayerFloats;

__global__ void __launch_bounds__(kThreads, 1)
trace_rev_kernel(const __grid_constant__ TraceRevArgs ra) {
  const TraceArgs& args = ra.t;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileCtx c = make_ctx(smem_raw);
  pipe_init(c.s);
  constexpr int T = 0, PTS = kTileRows;
  const long long count = args.active_in ? (long long)args.counters[args.iter] : args.P;
  const long long ntiles = (count + PTS - 1) / PTS;
  Pipe cp{0, 0};
  Prod prod;
  program_begin(c.s);
  program_add_fwd(c.s, args.sdf);
  if (args.has_dnet) program_add_fwd(c.s, args.dnet);
  if (args.do_update) {
    program_add_bwd(c.s, args.sdf);
    if (args.has_dnet) program_add_bwd(c.s, args.dnet);
  }
  prod.init(blockIdx.x, ntiles, gridDim.x);
  prod.prefill(c.s);
  float* ds_sdf = ra.scratch + (size_t)blockIdx.x * kScratchPerCta;
  float* ds_def = ds_sdf + (size_t)SR_MLP_MAX_LAYERS * kDstashLayerFloats;
  const int warp = threadIdx.x >> 5;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    load_points<T>(c, tile, count, args.active_in, args.pts, args.batch_inds, 0);
    consumer_sync();
    // ---- forward sweeps
    prologue_pe<T>(c, args.sdf, nullptr, 0);
    {
      const LastOut lo{nullptr, 0, c.row_pt, args.do_update ? ds_sdf : nullptr};
      run_net<T>(args.sdf, c.s, cp, prod, lo);
    }
    sdf_finish<T>(c);
    consumer_sync();
    if (args.has_dnet) {
      prologue_pe<T>(c, args.dnet, args.conds, args.condlen);
      const LastOut lo{nullptr, 0, c.row_pt, args.do_update ? ds_def : nullptr};
      run_net<T>(args.dnet, c.s, cp, prod, lo);
      deform_finish<T>(c, args.has_lbs ? &args.lbs : nullptr);
    } else {
      identity_deform<T>(c);
    }
    consumer_sync();
    // ---- test, loss, cotangents (one thread per ray)
    if (threadIdx.x < PTS) {
      float* a = c.aux + threadIdx.x * kAuxStride;
      const int gp = __float_as_int(a[AUX_GP]);
      float cot_f = 0.f, u[3] = {0.f, 0.f, 0.f}, loss = 0.f;
      int state = 0;  // 0: padding / done, 1: needs update
      if (gp >= 0) {
        const float f = a[AUX_F];
        const RayTest r = ray_test(f, a + AUX_D, args.rays + (size_t)gp * 3, args.tp);
        if (r.done) {
          args.converged[gp] = 1;
        } else if (args.do_update) {
          state = 1;
          loss = ray_loss(r, f, a + AUX_J, args.tp, u);
          cot_f = sdf_cotangent(f, args.tp);
        }
      }
      a[AUX_F] = cot_f;                 // slots reused: cotangent of f
      a[AUX_D] = u[0]; a[AUX_D + 1] = u[1]; a[AUX_D + 2] = u[2];
      a[AUX_OFF] = loss;
      a[AUX_OFF + 1] = __int_as_float(state);
    }
    consumer_sync();
    if (args.do_update) {
      // ---- backward sweep through the SDF: cotangent w1*sign(f) on output 0
      {
        const int kp = bwd_kpad(args.sdf.layer[args.sdf.n_layers - 1]);
        for (int idx = threadIdx.x; idx < kp * kTileRows; idx += kConsumerThreads) {
          const int k = idx / kTileRows, row = idx % kTileRows;
          c.s.at[(size_t)k * kRowStride + row] = (k == 0) ? c.aux[row * kAuxStride + AUX_F] : 0.f;
        }
        bwd_clear_stash(c.s);
        run_net_bwd(args.sdf, c.s, cp, prod, ds_sdf);  // epilogues carry the barriers
      }
      if (threadIdx.x < PTS) {
        float* a = c.aux + threadIdx.x * kAuxStride;
        const float x[3] = {a[AUX_P], a[AUX_P + 1], a[AUX_P + 2]};
        float g[3];
        embed_backward(c.s.at, threadIdx.x, x, args.sdf.multires, args.sdf.pe_w, g);
        a[AUX_GF] = g[0]; a[AUX_GF + 1] = g[1]; a[AUX_GF + 2] = g[2];
      }
      consumer_sync();
      // ---- backward sweep through the translator: cotangent u on its 3 outputs
      if (args.has_dnet) {
        const int kp = bwd_kpad(args.dnet.layer[args.dnet.n_layers - 1]);
        for (int idx = threadIdx.x; idx < kp * kTileRows; idx += kConsumerThreads) {
          const int k = idx / kTileRows, row = idx % kTileRows;
          c.s.at[(size_t)k * kRowStride + row] = (k < 3) ? c.aux[row * kAuxStride + AUX_D + k] : 0.f;
        }
        bwd_clear_stash(c.s);
        run_net_bwd(args.dnet, c.s, cp, prod, ds_def);
      }
      if (threadIdx.x < PTS) {
        float* a = c.aux + threadIdx.x * kAuxStride;
        const int gp = __float_as_int(a[AUX_GP]);
        if (gp >= 0 && __float_as_int(a[AUX_OFF + 1]) == 1) {
          const float x[3] = {a[AUX_P], a[AUX_P + 1], a[AUX_P + 2]};
          float g[3] = {a[AUX_GF] + a[AUX_D], a[AUX_GF + 1] + a[AUX_D + 1], a[AUX_GF + 2] + a[AUX_D + 2]};
          if (args.has_dnet) {
            float gd[3];
            embed_backward(c.s.at, threadIdx.x, x, args.dnet.multires, args.dnet.pe_w, gd);
            g[0] += gd[0]; g[1] += gd[1]; g[2] += gd[2];
          }
          newton_step(args.pts + (size_t)gp * 3, x, g, a[AUX_OFF], &args.counters[args.iter + 1], args.active_out,
                      gp);
        }
      }
    }
    consumer_sync();
  }
  (void)warp;
}

// ---------------------------------------------------------------------------------------------
// Shading geometry at surface points (infer path).
// ---------------------------------------------------------------------------------------------
struct ShadeArgs {
  sr_mlp_desc sdf;
  sr_mlp_desc dnet;
  sr_lbs_params lbs;
  int has_lbs;
  int has_dnet;
  const float* pts;
  const float* rays;
  const int64_t* batch_inds;
  const float* conds;
  int condlen;
  long long P;
  float* normals;
  float* crays;
  float* feat;
  int nfeat;
  float* dpos;
  uint8_t* inv_ok;
};

__global__ void __launch_bounds__(kThreads, 1)
shade_kernel(const __grid_constant__ ShadeArgs args) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileCtx c = make_ctx(smem_raw);
  pipe_init(c.s);
  constexpr int T = 3, PTS = kTileRows / (T + 1);
  const long long ntiles = (args.P + PTS - 1) / PTS;
  Pipe cp{0, 0};
  Prod prod;
  program_begin(c.s);
  program_add_fwd(c.s, args.sdf);
  if (args.has_dnet) program_add_fwd(c.s, args.dnet);
  prod.init(blockIdx.x, ntiles, gridDim.x);
  prod.prefill(c.s);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    load_points<T>(c, tile, args.P, nullptr, args.pts, args.batch_inds, 0);
    consumer_sync();
    prologue_pe<T>(c, args.sdf, nullptr, 0);
    {
      const LastOut lo{args.feat, args.nfeat, c.row_pt, nullptr};
      run_net<T>(args.sdf, c.s, cp, prod, lo);
    }
    sdf_finish<T>(c);
    consumer_sync();
    if (args.has_dnet) {
      prologue_pe<T>(c, args.dnet, args.conds, args.condlen);
      const LastOut lo{nullptr, 0, c.row_pt, nullptr};
      run_net<T>(args.dnet, c.s, cp, prod, lo);
      deform_finish<T>(c, args.has_lbs ? &args.lbs : nullptr);
    } else {
      identity_deform<T>(c);
    }
    consumer_sync();
    if (threadIdx.x < PTS) {
      const float* a = c.aux + threadIdx.x * kAuxStride;
      const int gp = __float_as_int(a[AUX_GP]);
      if (gp >= 0) {
        const bool ok = shade_point(a + AUX_GF, a + AUX_J, args.rays + (size_t)gp * 3, args.normals + (size_t)gp * 3,
                                    args.crays + (size_t)gp * 3);
        if (args.dpos) {
#pragma unroll
          for (int j = 0; j < 3; ++j) args.dpos[(size_t)gp * 3 + j] = a[AUX_D + j];
        }
        if (args.inv_ok) args.inv_ok[gp] = ok ? 1 : 0;
      }
    }
    consumer_sync();
  }
}

// ---------------------------------------------------------------------------------------------
// Small helpers
// ---------------------------------------------------------------------------------------------
// weight-norm fold + transpose + pad: one warp per output row n.
__global__ void __launch_bounds__(256)
fold_kernel(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ b,
            int n, int k, int npad, int kpad, float* __restrict__ wt, float* __restrict__ bias,
            float* __restrict__ wb, int wb_rows, int wb_cols) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= npad) return;
  const int row = warp;
  float scale = 0.f;
  if (row < n) {
    if (g) {
      float ss = 0.f;
      for (int j = lane; j < k; j += 32) { const float x = v[(size_t)row * k + j]; ss = fmaf(x, x, ss); }
      ss = sr_warp_sum(ss);
      scale = g[row] / sqrtf(ss);
    } else scale = 1.0f;
  }
  for (int j = lane; j < kpad; j += 32) {
    float w = 0.f;
    if (row < n && j < k) w = g ? v[(size_t)row * k + j] * scale : v[(size_t)row * k + j];
    wt[(size_t)j * npad + row] = w;
    if (wb && row < wb_rows) wb[(size_t)row * wb_cols + j] = w;  // un-transposed copy (j < kpad <= wb_cols)
  }
  if (wb && row < wb_rows)
    for (int j = kpad + lane; j < wb_cols; j += 32) wb[(size_t)row * wb_cols + j] = 0.f;
  if (lane == 0) bias[row] = (row < n && b) ? b[row] : 0.f;
}

// batch_rodrigues + kinematic chain + init-pose product; one thread per frame.
__global__ void bone_kernel(const float* __restrict__ poses, const float* __restrict__ Js,
                            const int32_t* __restrict__ parents, const float* __restrict__ ipi,
                            int F, float* __restrict__ A, float* __restrict__ posedJ) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  float res[24][12];  // rows 0..2 of each 4x4 (row 3 is 0 0 0 1)
  for (int i = 0; i < 24; ++i) {
    // batch_rodrigues (smpl_pytorch/util.py:35-46): norm of (theta + 1e-8)
    const float tx = poses[((size_t)f * 24 + i) * 3], ty = poses[((size_t)f * 24 + i) * 3 + 1],
                tz = poses[((size_t)f * 24 + i) * 3 + 2];
    const float ex = tx + 1e-8f, ey = ty + 1e-8f, ez = tz + 1e-8f;
    const float angle = sqrtf(ex * ex + ey * ey + ez * ez);
    const float nx = tx / angle, ny = ty / angle, nz = tz / angle;
    const float half = angle * 0.5f;
    const float vc = cosf(half), vs = sinf(half);
    float qw = vc, qx = vs * nx, qy = vs * ny, qz = vs * nz;
    // quat2mat (:48-68) renormalises
    const float qn = sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
    qw /= qn; qx /= qn; qy /= qn; qz /= qn;
    const float w2 = qw * qw, x2 = qx * qx, y2 = qy * qy, z2 = qz * qz;
    const float wx = qw * qx, wy = qw * qy, wz = qw * qz, xy = qx * qy, xz = qx * qz, yz = qy * qz;
    float R[9] = {w2 + x2 - y2 - z2, 2 * xy - 2 * wz, 2 * wy + 2 * xz,
                  2 * wz + 2 * xy, w2 - x2 + y2 - z2, 2 * yz - 2 * wx,
                  2 * xz - 2 * wy, 2 * wx + 2 * yz, w2 - x2 - y2 + z2};
    float t[3];
    const int par = i == 0 ? -1 : parents[i];
    for (int j = 0; j < 3; ++j) t[j] = i == 0 ? Js[j] : Js[i * 3 + j] - Js[par * 3 + j];
    if (i == 0) {
      for (int r = 0; r < 3; ++r) {
        for (int cc = 0; cc < 3; ++cc) res[0][4 * r + cc] = R[3 * r + cc];
        res[0][4 * r + 3] = t[r];
      }
    } else {
      const float* Pm = res[par];
      for (int r = 0; r < 3; ++r) {
        for (int cc = 0; cc < 3; ++cc)
          res[i][4 * r + cc] = Pm[4 * r] * R[cc] + Pm[4 * r + 1] * R[3 + cc] + Pm[4 * r + 2] * R[6 + cc];
        res[i][4 * r + 3] = Pm[4 * r] * t[0] + Pm[4 * r + 1] * t[1] + Pm[4 * r + 2] * t[2] + Pm[4 * r + 3];
      }
    }
  }
  for (int i = 0; i < 24; ++i) {
    float* out = A + ((size_t)f * 24 + i) * 16;
    if (posedJ) {
      for (int r = 0; r < 3; ++r) posedJ[((size_t)f * 24 + i) * 3 + r] = res[i][4 * r + 3];
    }
    if (ipi) {
      const float* Bm = ipi + (size_t)i * 16;
      for (int r = 0; r < 3; ++r)
        for (int cc = 0; cc < 4; ++cc)
          out[4 * r + cc] = res[i][4 * r] * Bm[cc] + res[i][4 * r + 1] * Bm[4 + cc] +
                            res[i][4 * r + 2] * Bm[8 + cc] + res[i][4 * r + 3] * Bm[12 + cc];
    } else {
      // A = results - pad(results @ [J;0])   (model/Deformer.py:196-200)
      for (int r = 0; r < 3; ++r) {
        const float ib = res[i][4 * r] * Js[i * 3] + res[i][4 * r + 1] * Js[i * 3 + 1] +
                         res[i][4 * r + 2] * Js[i * 3 + 2];
        for (int cc = 0; cc < 3; ++cc) out[4 * r + cc] = res[i][4 * r + cc];
        out[4 * r + 3] = res[i][4 * r + 3] - ib;
      }
    }
    out[12] = 0.f; out[13] = 0.f; out[14] = 0.f; out[15] = ipi ? 1.f : 1.f;
  }
}

// NCDHW [24][D*H*W] -> [D*H*W][24] through a shared-memory transpose (coalesced both ways).
__global__ void __launch_bounds__(256)
ws_to_cl_kernel(const float* __restrict__ src, float* __restrict__ dst, long long nvox) {
  __shared__ float tile[24][257];
  const long long v0 = (long long)blockIdx.x * 256;
  for (int ch = 0; ch < 24; ++ch) {
    const long long v = v0 + threadIdx.x;
    tile[ch][threadIdx.x] = v < nvox ? src[(size_t)ch * nvox + v] : 0.f;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 256 * 24; idx += 256) {
    const int vl = idx / 24, ch = idx % 24;
    if (v0 + vl < nvox) dst[(size_t)(v0 + vl) * 24 + ch] = tile[ch][vl];
  }
}

// ---------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------
int validate_net(const sr_mlp_desc* net, int T) {
  if (!net || net->n_layers < 1 || net->n_layers > SR_MLP_MAX_LAYERS) return SR_EINVAL;
  if (net->multires < 0 || net->multires > 16) return SR_EINVAL;
  for (int l = 0; l < net->n_layers; ++l) {
    const sr_mlp_layer& L = net->layer[l];
    if (!L.wt || !L.bias) return SR_EINVAL;
    if (L.kpad % kKT || L.kpad < kKT || L.kpad > kMaxK || L.k > L.kpad) return SR_EUNSUPPORTED;
    if (L.npad % 128 || L.npad < 128 || L.npad > kMaxN || L.n > L.npad) return SR_EUNSUPPORTED;
    if (l > 0) {
      const int expect = net->layer[l - 1].n + (L.skip ? net->d_in : 0);
      if (L.k != expect) return SR_EINVAL;
      if (L.skip && net->d_in > kStashMax) return SR_EUNSUPPORTED;
    } else if (L.k != net->d_in || L.skip) return SR_EINVAL;
  }
  (void)T;
  return SR_OK;
}

// ---------------------------------------------------------------------------------------------
// Small-batch fp32 evaluation of the SDF value for a LIST of points (sign / threshold decisions on the few values the
// tensor-core engine leaves inside its error band).  The persistent engine above is throughput-shaped: one CTA walks
// all layers of a 64-row tile, the same latency however few points there are.  Here every layer is one launch whose
// CTAs split the COLUMNS (64 per CTA) and a group of 8 listed points, so a handful of points uses the whole GPU
// (9 short launches).  Plain fp32 FMAs in k order; activations fp32 in global scratch [cap][512] x 2.
// ---------------------------------------------------------------------------------------------
constexpr int kSmallPts = 8;     // listed points per CTA
constexpr int kSmallCols = 64;   // output columns per CTA

__global__ void __launch_bounds__(256)
small_embed_kernel(const float* __restrict__ pts, const int32_t* __restrict__ index, const int32_t* __restrict__ m_dev,
                   int cap, int multires, sr_mlp_desc net, float* __restrict__ emb, int ld) {
  const int count = min(*m_dev, cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const int gp = index[i];
  float* e = emb + (size_t)i * ld;
  float freq = 1.0f;
#pragma unroll
  for (int j = 0; j < 3; ++j) e[j] = pts[(size_t)gp * 3 + j];
  for (int b = 0; b < multires; ++b, freq *= 2.0f) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float sn, cs;
      sincosf(pts[(size_t)gp * 3 + j] * freq, &sn, &cs);
      e[3 + 6 * b + j] = net.pe_w[b] * sn;
      e[6 + 6 * b + j] = net.pe_w[b] * cs;
    }
  }
}

struct SmallLayerArgs {
  const float* wt;      // [kpad][npad] k-major folded weights
  const float* bias;
  int k, n, npad, act;
  const float* in;      // [cap][ld_in] (previous activations or the embedding)
  int ld_in, k_in;      // columns taken from `in`
  const float* emb;     // skip source [cap][ld_emb] (or null): input = cat(in[:k_in], emb[:k - k_in]) * scale
  int ld_emb;
  float scale;
  float* out;           // [cap][ld_out] (or null on the last layer)
  int ld_out;
  float* sdf;           // last layer: sdf[index[i]] = output column 0
  const int32_t* index;
  const int32_t* m_dev;
  int cap;
};

__global__ void __launch_bounds__(256) small_layer_kernel(const __grid_constant__ SmallLayerArgs a) {
  const int count = min(*a.m_dev, a.cap);
  const int p0 = blockIdx.y * kSmallPts;
  if (p0 >= count) return;
  __shared__ float xs[kSmallPts][512];
  const int np = min(kSmallPts, count - p0);
  const int k8s = (a.k + 7) & ~7;
  for (int idx = threadIdx.x; idx < kSmallPts * k8s; idx += blockDim.x) {
    const int p = idx / k8s, k = idx % k8s;
    float v = 0.f;
    if (p < np && k < a.k) {
      const size_t row = (size_t)(p0 + p);
      v = k < a.k_in ? a.in[row * a.ld_in + k] : a.emb[row * a.ld_emb + (k - a.k_in)];
      v *= a.scale;
    }
    xs[p][k] = v;
  }
  __syncthreads();
  const int col = blockIdx.x * kSmallCols + (threadIdx.x & (kSmallCols - 1));
  const int pg = threadIdx.x / kSmallCols;            // 4 point pairs
  if (col >= a.n) return;
  float acc0 = 0.f, acc1 = 0.f;
  const float* w = a.wt + col;
  const float* x0 = xs[2 * pg];
  const float* x1 = xs[2 * pg + 1];
  // the folded weights are zero padded to kpad (a multiple of 8) rows: 8 loads in flight per step, FMAs in k order
  const int k8 = (a.k + 7) & ~7;
  for (int k = 0; k < k8; k += 8) {
    float wv[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) wv[u] = __ldg(w + (size_t)(k + u) * a.npad);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      acc0 = fmaf(x0[k + u], wv[u], acc0);
      acc1 = fmaf(x1[k + u], wv[u], acc1);
    }
  }
  const float b = a.bias[col];
  float z[2] = {acc0 + b, acc1 + b};
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int p = 2 * pg + t;
    if (p >= np) continue;
    float v = z[t];
    if (a.act == SR_ACT_SOFTPLUS100) { float d; v = softplus100(v, d); }
    else if (a.act == SR_ACT_RELU) v = fmaxf(v, 0.f);
    else if (a.act == SR_ACT_TANH) v = tanhf(v);
    if (a.out) a.out[(size_t)(p0 + p) * a.ld_out + col] = v;
    if (a.sdf && col == 0) a.sdf[a.index[p0 + p]] = v;
  }
}

// ids of the values within eps of `center` -> list (warp-aggregated append; order is irrelevant
// to the caller, which writes results back by id)
__global__ void __launch_bounds__(256)
band_select_kernel(const float* __restrict__ v, long long n, float center, float eps,
                   int32_t* __restrict__ list, int32_t* __restrict__ counter) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n_round = (n + 31) / 32 * 32;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    const bool hit = i < n && fabsf(v[i] - center) < eps;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (m == 0u) continue;
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == 0) base = atomicAdd(counter, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (hit) list[base + __popc(m & ((1u << lane) - 1u))] = (int32_t)i;
  }
}

template <typename K>
int set_smem(K kernel) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)kDynSmem);
  return e == cudaSuccess ? SR_OK : (int)e;
}

int grid_for_tiles(long long ntiles) {
  return (int)(ntiles < SR_NUM_SMS ? (ntiles < 1 ? 1 : ntiles) : SR_NUM_SMS);
}

}  // namespace

extern "C" {

int sr_fold_linear(const float* v, const float* g, const float* b, int n, int k, int npad,
                   int kpad, float* wt, float* bias_out, float* wb, cudaStream_t s) {
  if (!v || !wt || !bias_out || n <= 0 || k <= 0 || npad < n || kpad < k) return SR_EINVAL;
  const int warps_per_block = 8;
  const int wb_rows = (n + kKT - 1) / kKT * kKT, wb_cols = (k + 127) / 128 * 128;
  if (wb_rows > npad) return SR_EINVAL;
  fold_kernel<<<sr_div_up(npad, warps_per_block), 256, 0, s>>>(v, g, b, n, k, npad, kpad, wt,
                                                               bias_out, wb, wb_rows, wb_cols);
  return sr_launch_status();
}

int sr_sdf_forward(const sr_mlp_desc* net, const float* pts, int64_t P, float* sdf, float* grad,
                   float* feat, int nfeat, cudaStream_t s) {
  int rc = validate_net(net, grad ? 3 : 0);
  if (rc) return rc;
  if (P < 0 || P > 0x7fffffffLL) return SR_EINVAL;
  if (P == 0) return SR_OK;
  if (!pts || !sdf) return SR_EINVAL;
  if (net->d_in != 3 + 6 * net->multires) return SR_EINVAL;
  if (feat && (nfeat <= 0 || nfeat + 1 > net->layer[net->n_layers - 1].n)) return SR_EINVAL;
  SdfArgs a;
  a.net = *net; a.pts = pts; a.P = P; a.sdf = sdf; a.grad = grad; a.feat = feat; a.nfeat = nfeat;
  a.index = nullptr; a.m_dev = nullptr;
  if (grad) {
    if ((rc = set_smem(sdf_kernel<3>))) return rc;
    const long long nt = (P + 15) / 16;
    sdf_kernel<3><<<grid_for_tiles(nt), kThreads, kDynSmem, s>>>(a);
  } else {
    if ((rc = set_smem(sdf_kernel<0>))) return rc;
    const long long nt = (P + 63) / 64;
    sdf_kernel<0><<<grid_for_tiles(nt), kThreads, kDynSmem, s>>>(a);
  }
  return sr_launch_status();
}

// Value-only re-evaluation of the points listed in `index` (device-side count `m_dev`, at most P)
// on this fp32 engine; sdf[index[i]] is overwritten.  Used to decide signs / thresholds of values
// the tensor-core engine left inside its error band (MCAcc/seg3d_lossless.py:333-346 compares
// `> balance`; utils/FindSurfacePs.py:120-127 compares `< dthreshold`).
int sr_sdf_forward_indexed(const sr_mlp_desc* net, const float* pts, int64_t P, const int32_t* index,
                           const int32_t* m_dev, float* sdf, cudaStream_t s) {
  int rc = validate_net(net, 0);
  if (rc) return rc;
  if (P < 0 || P > 0x7fffffffLL) return SR_EINVAL;
  if (P == 0) return SR_OK;
  if (!pts || !sdf || !index || !m_dev) return SR_EINVAL;
  if (net->d_in != 3 + 6 * net->multires) return SR_EINVAL;
  SdfArgs a;
  a.net = *net; a.pts = pts; a.P = P; a.sdf = sdf; a.grad = nullptr; a.feat = nullptr; a.nfeat = 0;
  a.index = index; a.m_dev = m_dev;
  if ((rc = set_smem(sdf_kernel<0>))) return rc;
  const long long nt = (P + 63) / 64;
  sdf_kernel<0><<<grid_for_tiles(nt), kThreads, kDynSmem, s>>>(a);
  return sr_launch_status();
}

int64_t sr_sdf_small_work_bytes(int cap) { return (int64_t)cap * (2 * 512 + 64) * 4; }

// Value-only fp32 evaluation of the listed points with column-split launches (low latency for short lists); the
// first `cap` entries of the list are handled here, the rest (if the list is longer) by the persistent engine.
int sr_sdf_forward_small(const sr_mlp_desc* net, const float* pts, int64_t P, const int32_t* index, const int32_t* m_dev,
                         float* sdf, void* work, int cap, cudaStream_t s) {
  int rc = validate_net(net, 0);
  if (rc) return rc;
  if (P <= 0 || P > 0x7fffffffLL || !pts || !sdf || !index || !m_dev || !work || cap <= 0) return SR_EINVAL;
  if (net->d_in != 3 + 6 * net->multires || net->d_in > 64) return SR_EINVAL;
  float* emb = (float*)work;
  float* bufs[2] = {emb + (size_t)cap * 64, emb + (size_t)cap * (64 + 512)};
  small_embed_kernel<<<(cap + 255) / 256, 256, 0, s>>>(pts, index, m_dev, cap, net->multires, *net, emb, 64);
  const float* in = emb;
  int ld_in = 64, k_prev = net->d_in;
  for (int l = 0; l < net->n_layers; ++l) {
    const sr_mlp_layer& ly = net->layer[l];
    if (ly.k > 512 || ly.n > 512) return SR_EUNSUPPORTED;
    SmallLayerArgs a;
    a.wt = ly.wt; a.bias = ly.bias; a.k = ly.k; a.n = ly.n; a.npad = ly.npad; a.act = ly.act;
    a.in = in; a.ld_in = ld_in;
    a.k_in = ly.skip ? ly.k - net->d_in : ly.k;
    a.emb = ly.skip ? emb : nullptr; a.ld_emb = 64;
    a.scale = ly.skip ? 0.70710678118654752440f : 1.0f;
    const bool last = l == net->n_layers - 1;
    a.out = last ? nullptr : bufs[l & 1]; a.ld_out = 512;
    a.sdf = last ? sdf : nullptr; a.index = index; a.m_dev = m_dev; a.cap = cap;
    (void)k_prev;
    dim3 grid((ly.n + kSmallCols - 1) / kSmallCols, (cap + kSmallPts - 1) / kSmallPts);
    small_layer_kernel<<<grid, 256, 0, s>>>(a);
    in = bufs[l & 1]; ld_in = 512; k_prev = ly.n;
  }
  return sr_launch_status();
}

int sr_band_select(const float* values, int64_t n, float center, float eps, int32_t* list,
                   int32_t* counter, cudaStream_t s) {
  if (!values || !list || !counter || n < 0 || n > 0x7fffffffLL) return SR_EINVAL;
  if (n == 0) return SR_OK;
  band_select_kernel<<<sr_grid_for(n, 256, 8), 256, 0, s>>>(values, n, center, eps, list, counter);
  return sr_launch_status();
}

int sr_lbs_bone_transforms(const float* poses, const float* Js, const int32_t* parents,
                           const float* init_pose_inv, int F, float* A, float* posedJ,
                           cudaStream_t s) {
  if (F < 0 || !poses || !Js || !parents || !A) return SR_EINVAL;
  if (F == 0) return SR_OK;
  bone_kernel<<<sr_div_up(F, 32), 32, 0, s>>>(poses, Js, parents, init_pose_inv, F, A, posedJ);
  return sr_launch_status();
}

int sr_lbs_weights_to_channels_last(const float* ws_ncdhw, float* ws_cl, int D, int H, int W,
                                    cudaStream_t s) {
  if (!ws_ncdhw || !ws_cl || D <= 0 || H <= 0 || W <= 0) return SR_EINVAL;
  const long long nvox = (long long)D * H * W;
  ws_to_cl_kernel<<<sr_div_up(nvox, 256), 256, 0, s>>>(ws_ncdhw, ws_cl, nvox);
  return sr_launch_status();
}

static int check_lbs(const sr_lbs_params* lbs) {
  if (!lbs) return SR_OK;
  if (!lbs->ws_cl || !lbs->A || !lbs->trans || lbs->D <= 0 || lbs->H <= 0 || lbs->W <= 0 ||
      lbs->F <= 0)
    return SR_EINVAL;
  return SR_OK;
}

int sr_deform_forward(const sr_mlp_desc* net, const sr_lbs_params* lbs, const float* pts,
                      const int64_t* batch_inds, int64_t pts_per_frame, const float* conds,
                      int condlen, int64_t P, float* d, float* offset, float* jac,
                      int32_t* corner_idx, cudaStream_t s) {
  int rc = validate_net(net, jac ? 3 : 0);
  if (rc) return rc;
  if ((rc = check_lbs(lbs))) return rc;
  if (P < 0 || P > 0x7fffffffLL || condlen < 0) return SR_EINVAL;
  if (P == 0) return SR_OK;
  if (!pts || !d || (condlen > 0 && !conds)) return SR_EINVAL;
  if (net->d_in != 3 + 6 * net->multires + condlen) return SR_EINVAL;
  if (net->layer[net->n_layers - 1].n != 3) return SR_EINVAL;
  DeformArgs a;
  a.net = *net;
  a.has_lbs = lbs ? 1 : 0;
  if (lbs) a.lbs = *lbs;
  a.pts = pts; a.batch_inds = batch_inds; a.pts_per_frame = pts_per_frame; a.conds = conds;
  a.condlen = condlen; a.P = P; a.d = d; a.offset = offset; a.jac = jac; a.corner_idx = corner_idx;
  if (jac) {
    if ((rc = set_smem(deform_kernel<3>))) return rc;
    deform_kernel<3><<<grid_for_tiles((P + 15) / 16), kThreads, kDynSmem, s>>>(a);
  } else {
    if ((rc = set_smem(deform_kernel<0>))) return rc;
    deform_kernel<0><<<grid_for_tiles((P + 63) / 64), kThreads, kDynSmem, s>>>(a);
  }
  return sr_launch_status();
}

int sr_render_forward(const sr_mlp_desc* net, const float* pts, const float* normals,
                      const float* views, const float* feat, int nfeat, int64_t P, float* rgb,
                      cudaStream_t s) {
  int rc = validate_net(net, 0);
  if (rc) return rc;
  if (P < 0 || P > 0x7fffffffLL || nfeat < 0) return SR_EINVAL;
  if (P == 0) return SR_OK;
  if (!pts || !normals || !views || !rgb || (nfeat > 0 && !feat)) return SR_EINVAL;
  if (net->d_in != 3 + (3 + 6 * net->multires) + 3 + nfeat) return SR_EINVAL;
  if (net->layer[net->n_layers - 1].n > 8) return SR_EUNSUPPORTED;
  RenderArgs a;
  a.net = *net; a.pts = pts; a.normals = normals; a.views = views; a.feat = feat; a.nfeat = nfeat;
  a.P = P; a.rgb = rgb;
  if ((rc = set_smem(render_kernel))) return rc;
  render_kernel<<<grid_for_tiles((P + 63) / 64), kThreads, kDynSmem, s>>>(a);
  return sr_launch_status();
}

int sr_trace_step(const sr_mlp_desc* sdf, const sr_mlp_desc* dnet, const sr_lbs_params* lbs,
                  const sr_trace_params* tp, float* pts, const float* rays,
                  const int64_t* batch_inds, const float* conds, int condlen, int64_t P,
                  const int32_t* active_in, int32_t* active_out, int32_t* counters, int iter,
                  uint8_t* converged, cudaStream_t s) {
  int rc = validate_net(sdf, 3);
  if (rc) return rc;
  if (dnet && (rc = validate_net(dnet, 3))) return rc;
  if (!dnet && lbs) return SR_EINVAL;
  if ((rc = check_lbs(lbs))) return rc;
  if (!tp || P < 0 || P > 0x7fffffffLL || iter < 0) return SR_EINVAL;
  if (P == 0) return SR_OK;
  if (!pts || !rays || !counters || !converged) return SR_EINVAL;
  if (sdf->d_in != 3 + 6 * sdf->multires) return SR_EINVAL;
  if (dnet && dnet->d_in != 3 + 6 * dnet->multires + condlen) return SR_EINVAL;
  if (dnet && dnet->layer[dnet->n_layers - 1].n != 3) return SR_EINVAL;
  TraceArgs a;
  a.sdf = *sdf;
  a.has_dnet = dnet ? 1 : 0;
  if (dnet) a.dnet = *dnet;
  a.has_lbs = lbs ? 1 : 0;
  if (lbs) a.lbs = *lbs;
  a.tp = *tp; a.pts = pts; a.rays = rays; a.batch_inds = batch_inds; a.conds = conds;
  a.condlen = condlen; a.P = P; a.active_in = active_in; a.active_out = active_out;
  a.counters = counters; a.iter = iter; a.do_update = active_out ? 1 : 0; a.converged = converged;
  if ((rc = set_smem(trace_kernel))) return rc;
  const long long nt = (P + 15) / 16;
  trace_kernel<<<grid_for_tiles(nt), kThreads, kDynSmem, s>>>(a);
  return sr_launch_status();
}

int64_t sr_trace_scratch_bytes(void) {
  return (int64_t)SR_NUM_SMS * (int64_t)kScratchPerCta * (int64_t)sizeof(float);
}

int sr_trace_step_rev(const sr_mlp_desc* sdf, const sr_mlp_desc* dnet, const sr_lbs_params* lbs,
                      const sr_trace_params* tp, float* pts, const float* rays,
                      const int64_t* batch_inds, const float* conds, int condlen, int64_t P,
                      const int32_t* active_in, int32_t* active_out, int32_t* counters, int iter,
                      uint8_t* converged, float* scratch, cudaStream_t s) {
  int rc = validate_net(sdf, 0);
  if (rc) return rc;
  if (dnet && (rc = validate_net(dnet, 0))) return rc;
  if (!dnet && lbs) return SR_EINVAL;
  if ((rc = check_lbs(lbs))) return rc;
  if (!tp || P < 0 || P > 0x7fffffffLL || iter < 0) return SR_EINVAL;
  if (P == 0) return SR_OK;
  if (!pts || !rays || !counters || !converged || !scratch) return SR_EINVAL;
  if (sdf->d_in != 3 + 6 * sdf->multires) return SR_EINVAL;
  if (dnet && dnet->d_in != 3 + 6 * dnet->multires + condlen) return SR_EINVAL;
  if (dnet && dnet->layer[dnet->n_layers - 1].n != 3) return SR_EINVAL;
  for (int l = 0; l < sdf->n_layers; ++l)
    if (!sdf->layer[l].wb) return SR_EINVAL;
  if (dnet)
    for (int l = 0; l < dnet->n_layers; ++l)
      if (!dnet->layer[l].wb) return SR_EINVAL;
  TraceRevArgs a;
  a.t.sdf = *sdf;
  a.t.has_dnet = dnet ? 1 : 0;
  if (dnet) a.t.dnet = *dnet;
  a.t.has_lbs = lbs ? 1 : 0;
  if (lbs) a.t.lbs = *lbs;
  a.t.tp = *tp; a.t.pts = pts; a.t.rays = rays; a.t.batch_inds = batch_inds; a.t.conds = conds;
  a.t.condlen = condlen; a.t.P = P; a.t.active_in = active_in; a.t.active_out = active_out;
  a.t.counters = counters; a.t.iter = iter; a.t.do_update = active_out ? 1 : 0;
  a.t.converged = converged;
  a.scratch = scratch;
  if ((rc = set_smem(trace_rev_kernel))) return rc;
  const long long nt = (P + kTileRows - 1) / kTileRows;
  trace_rev_kernel<<<grid_for_tiles(nt), kThreads, kDynSmem, s>>>(a);
  return sr_launch_status();
}

int sr_shade_geometry(const sr_mlp_desc* sdf, const sr_mlp_desc* dnet, const sr_lbs_params* lbs,
                      const float* pts, const float* rays, const int64_t* batch_inds,
                      const float* conds, int condlen, int64_t P, float* normals, float* crays,
                      float* feat, int nfeat, float* dpos, uint8_t* inv_ok, cudaStream_t s) {
  int rc = validate_net(sdf, 3);
  if (rc) return rc;
  if (dnet && (rc = validate_net(dnet, 3))) return rc;
  if (!dnet && lbs) return SR_EINVAL;
  if ((rc = check_lbs(lbs))) return rc;
  if (P < 0 || P > 0x7fffffffLL) return SR_EINVAL;
  if (P == 0) return SR_OK;
  if (!pts || !rays || !normals || !crays) return SR_EINVAL;
  if (sdf->d_in != 3 + 6 * sdf->multires) return SR_EINVAL;
  if (dnet && dnet->d_in != 3 + 6 * dnet->multires + condlen) return SR_EINVAL;
  if (feat && (nfeat <= 0 || nfeat + 1 > sdf->layer[sdf->n_layers - 1].n)) return SR_EINVAL;
  ShadeArgs a;
  a.sdf = *sdf;
  a.has_dnet = dnet ? 1 : 0;
  if (dnet) a.dnet = *dnet;
  a.has_lbs = lbs ? 1 : 0;
  if (lbs) a.lbs = *lbs;
  a.pts = pts; a.rays = rays; a.batch_inds = batch_inds; a.conds = conds; a.condlen = condlen;
  a.P = P; a.normals = normals; a.crays = crays; a.feat = feat; a.nfeat = nfeat; a.dpos = dpos;
  a.inv_ok = inv_ok;
  if ((rc = set_smem(shade_kernel))) return rc;
  shade_kernel<<<grid_for_tiles((P + 15) / 16), kThreads, kDynSmem, s>>>(a);
  return sr_launch_status();
}

int sr_abi_version(void) { return 1; }
const char* sr_build_info(void) { return "selfrecon_b200 sm_90a fp32-ffma-fused " __DATE__; }
}
