/*
 * selfrecon_b200.h -- C ABI of libselfrecon_b200.so (H100 / sm_90a).
 *
 * This is the drop-in boundary for the SelfRecon per-frame optimisation hot path
 * (SURVEY.md section 8).  Every entry point takes plain device pointers, sizes and a
 * cudaStream_t; none allocates, none synchronises the host, none touches torch types.
 * Each returns SR_OK (0), a negative SR_E* validation code, or a positive cudaError_t
 * raised by the launch.  The torch-facing shims (selfreconcode_b200/dropin/ *.py) own
 * allocation and turn non-zero codes into RuntimeError, mirroring the reference's pybind
 * modules FastMinv, MCGpu, GridSamplerMine, interp2x_boundary3d.
 *
 * Reference interface replaced by each group is cited as  <file>:<line>  relative to
 * jby1993/SelfReconCode.
 */
#ifndef SELFRECON_B200_H_
#define SELFRECON_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef __DRIVER_TYPES_H__
typedef struct CUstream_st* cudaStream_t;
#endif

enum {
  SR_OK = 0,
  SR_EINVAL = -1,     /* bad size / null pointer */
  SR_EUNSUPPORTED = -2, /* shape outside what the kernels are built for */
  SR_ECAPACITY = -3   /* caller-provided output buffer too small */
};

/* Library / build identification (used by the "loads and exports" CPU test). */
int sr_abi_version(void);
const char* sr_build_info(void);

/* ------------------------------------------------------------------------------------------
 * Batched 3x3 inverse + analytic backward.
 * Replaces FastMinv.Fast3x3Minv / Fast3x3Minv_backward
 *   (FastMinv/M3x3Inv.cpp:12-59, FastMinv/Matrix3x3InvKernels.cu:22-104).
 *   ms/invs/grads/outs: [n,3,3] contiguous; checks: [n] bytes (0/1, torch.bool layout).
 *   |det| < 1e-4  ->  inverse = 0, check = 0 (same threshold, compared in double as the
 *   reference's `fabs(det)<0.0001` does).
 * ------------------------------------------------------------------------------------------ */
int sr_minv3x3_f32(const float* ms, float* invs, uint8_t* checks, int64_t n, cudaStream_t s);
int sr_minv3x3_f64(const double* ms, double* invs, uint8_t* checks, int64_t n, cudaStream_t s);
int sr_minv3x3_bwd_f32(const float* grads, const float* invs, float* outs, int64_t n,
                       cudaStream_t s);
int sr_minv3x3_bwd_f64(const double* grads, const double* invs, double* outs, int64_t n,
                       cudaStream_t s);

/* ------------------------------------------------------------------------------------------
 * Marching cubes over a dense SDF grid, shared-vertex indexing, deterministic order.
 * Replaces MCGpu.mc_gpu (MCGpu/MCGpu.cpp:20-56, MCGpu/CudaKernels.cu:304-521,620-640).
 *   sdf: [nx,ny,nz] contiguous f32, index (i*ny + j)*nz + k; inside = sdf < iso.
 * Two calls (the reference also has one blocking readback of its two counters,
 * CudaKernels.cu:628):
 *   sr_mc_count : classify pass.  Fills `work` (sr_mc_work_bytes(nx,ny,nz) bytes, caller
 *                 allocated, kept until sr_mc_emit) and writes counts[0]=#vertices,
 *                 counts[1]=#faces on the device.
 *   sr_mc_emit  : writes vertices[V,3] (world: fmaf(v,step,min) per axis) and faces[F,3]
 *                 int64 (winding reversed like d_conver_ijkd_to_pindex) in CANONICAL order:
 *                 vertices sorted by owning edge key (i,j,k,dir), faces by (voxel, tri#).
 *                 Corners that reference a never-created boundary-layer vertex get -1,
 *                 as in the reference.  `i_offset` (0 for a whole grid) is added to the x
 *                 voxel index before scaling, so an x-slab of a larger grid produces the
 *                 same bits as the whole-grid call (multi-GPU extraction).
 * ------------------------------------------------------------------------------------------ */
int64_t sr_mc_work_bytes(int nx, int ny, int nz);
int sr_mc_count(const float* sdf, int nx, int ny, int nz, float iso, void* work, int32_t* counts,
                cudaStream_t s);
int sr_mc_emit(const float* sdf, int nx, int ny, int nz, float iso, float xstep, float ystep,
               float zstep, float xmin, float ymin, float zmin, int i_offset, const void* work,
               float* vertices, int64_t vcap, int64_t* faces, int64_t fcap, cudaStream_t s);

/* ------------------------------------------------------------------------------------------
 * 2x-1 trilinear upsample + boundary flag.
 * Replaces interp2x_boundary3d.forward/backward
 *   (MCAcc/cuda/interp2x_boundary3d.cpp:17-36, interp2x_boundary3d_kernel.cu:10-239).
 *   in: [bc,d,h,w] -> out: [bc,2d-1,2h-1,2w-1]; is_boundary: bytes, same shape as out.
 * ------------------------------------------------------------------------------------------ */
int sr_interp2x3d_fwd_f32(const float* in, float* out, uint8_t* is_boundary, int bc, int d, int h,
                          int w, float balance, cudaStream_t s);
int sr_interp2x3d_bwd_f32(const float* grad_out, float* grad_in, int bc, int d, int h, int w,
                          cudaStream_t s);
/* 2-D analogue (MCAcc/cuda/interp2x_boundary2d.cpp:17-36); unused by the reference's Python. */
int sr_interp2x2d_fwd_f32(const float* in, float* out, uint8_t* is_boundary, int bc, int h, int w,
                          float balance, cudaStream_t s);
int sr_interp2x2d_bwd_f32(const float* grad_out, float* grad_in, int bc, int h, int w,
                          cudaStream_t s);

/* ------------------------------------------------------------------------------------------
 * Trilinear grid sampler, border padding, align_corners=False, with first and second
 * order backward.  Replaces GridSamplerMine.forward/backward/dbackward
 *   (MCAcc/cuda/GridSamplerMine.cpp:73-96, GridSamplerMineKernel.cu:160-914).
 *   input  : [N,C,D,H,W] with element strides istr[5]   (any strides)
 *   grid   : [N,P,3] contiguous (P = Do*Ho*Wo flattened)
 *   output / grad_output : [N,C,P] contiguous
 *   grad_input  : [N,C,D,H,W] contiguous, MUST be zero-filled by the caller (atomics)
 *   corner_idx (optional, may be NULL): [N,P,3] int32 = floor of the clipped
 *                 un-normalised coordinate (ix,iy,iz) -- the "skinning indices".
 * ------------------------------------------------------------------------------------------ */
int sr_grid_sample3d_fwd_f32(const float* input, const int64_t* istr, const float* grid,
                             float* output, int32_t* corner_idx, int N, int C, int D, int H, int W,
                             int64_t P, cudaStream_t s);
int sr_grid_sample3d_bwd_f32(const float* input, const int64_t* istr, const float* grid,
                             const float* grad_output, float* grad_input, float* grad_grid, int N,
                             int C, int D, int H, int W, int64_t P, cudaStream_t s);
int sr_grid_sample3d_dbwd_f32(const float* gg_input /*[N,C,D,H,W] contiguous*/,
                              const float* gg_grid /*[N,P,3]*/, const float* input,
                              const int64_t* istr, const float* grid, const float* grad_output,
                              float* grad_input /*zeroed*/, float* grad_grid,
                              float* grad_grad_output, int N, int C, int D, int H, int W,
                              int64_t P, cudaStream_t s);
int sr_grid_sample3d_fwd_f64(const double* input, const int64_t* istr, const double* grid,
                             double* output, int32_t* corner_idx, int N, int C, int D, int H,
                             int W, int64_t P, cudaStream_t s);
int sr_grid_sample3d_bwd_f64(const double* input, const int64_t* istr, const double* grid,
                             const double* grad_output, double* grad_input, double* grad_grid,
                             int N, int C, int D, int H, int W, int64_t P, cudaStream_t s);
int sr_grid_sample3d_dbwd_f64(const double* gg_input, const double* gg_grid, const double* input,
                              const int64_t* istr, const double* grid, const double* grad_output,
                              double* grad_input, double* grad_grid, double* grad_grad_output,
                              int N, int C, int D, int H, int W, int64_t P, cudaStream_t s);

/* ------------------------------------------------------------------------------------------
 * Fused MLP stacks (positional encoding + all layers + activations in one kernel).
 *
 * A network is described by an sr_mlp_desc living in HOST memory (copied by value at
 * launch).  Weights are passed pre-folded by sr_fold_linear: W_T[k][n] (k-major, n padded
 * to a multiple of 128, k padded to a multiple of 8, zero filled), bias[n].
 * Replaces ImplicitNetwork.forward/.gradient (model/network.py:72-114),
 * MLPTranslator.forward (model/Deformer.py:49-76),
 * RenderingNetwork_view_norm.forward (model/RenderNet.py:54-89) and the Embedder
 * (model/Embedder.py:34-55, utils/utils.py:40-46).
 * ------------------------------------------------------------------------------------------ */
#define SR_MLP_MAX_LAYERS 12
enum { SR_ACT_NONE = 0, SR_ACT_SOFTPLUS100 = 1, SR_ACT_RELU = 2, SR_ACT_TANH = 3 };

typedef struct sr_mlp_layer {
  const float* wt;   /* [kpad][npad] device */
  const float* bias; /* [npad] device */
  int k;             /* true fan-in (after skip concat) */
  int n;             /* true fan-out */
  int kpad;          /* multiple of 8, <= 512 */
  int npad;          /* multiple of 128, <= 512 */
  int act;           /* SR_ACT_* applied to this layer's output */
  int skip;          /* 1: input = cat([x, net_input]) / sqrt(2) (network.py:88-89) */
  const float* wb;   /* [pad8(n)][pad128(k)] device: un-transposed padded copy streamed by the
                        reverse-mode pass (may be NULL when only forward kernels are used) */
} sr_mlp_layer;

typedef struct sr_mlp_desc {
  int n_layers;
  int d_in;          /* width of the embedded network input (39 / 167 / 289 ...) */
  int multires;      /* PE bands on the 3-vector that is embedded */
  float pe_w[16];    /* per-band annealing weights (utils/utils.py:40-46), one per band */
  sr_mlp_layer layer[SR_MLP_MAX_LAYERS];
} sr_mlp_desc;

/* weight-norm fold + transpose + pad:  W = g * v / ||v||_row  (g == NULL -> W = v).
 *   v: [n,k] row-major (torch nn.Linear.weight), g: [n] or NULL, b: [n] or NULL.
 *   wt: [kpad][npad], bias_out: [npad].  (network.py:65-66, RenderNet.py:46-47) */
int sr_fold_linear(const float* v, const float* g, const float* b, int n, int k, int npad,
                   int kpad, float* wt, float* bias_out, float* wb /* [pad8(n)][pad128(k)] or NULL */,
                   cudaStream_t s);

/* SDF network.  pts [P,3] -> sdf[P]; optional grad[P,3] (= d sdf / d pts, forward-mode),
 * optional feat[P,nfeat] (outputs 1..nfeat of the last layer = `rendcond`).            */
int sr_sdf_forward(const sr_mlp_desc* net, const float* pts, int64_t P, float* sdf, float* grad,
                   float* feat, int nfeat, cudaStream_t s);

/* Per-frame bone transforms for LBS: axis-angle -> rotation (batch_rodrigues,
 * smpl_pytorch/util.py:35-68), kinematic chain and init-pose product
 * (model/Deformer.py:176-203).  poses [F,24,3], Js [24,3], parents [24] int32,
 * init_pose_inv [24,4,4] (or NULL: Deformer.py:196-200 branch) -> A [F,24,4,4].          */
int sr_lbs_bone_transforms(const float* poses, const float* Js, const int32_t* parents,
                           const float* init_pose_inv, int F, float* A, float* posedJ /*[F,24,3] or NULL*/,
                           cudaStream_t s);

typedef struct sr_lbs_params {
  const float* ws_cl;   /* skin-weight volume, channels-last [D,H,W,24] device */
  int D, H, W;
  float bmin[3], bmax[3];
  const float* A;       /* [F,24,4,4] from sr_lbs_bone_transforms */
  const float* trans;   /* [F,3] */
  int F;
} sr_lbs_params;

/* NCDHW [1,24,D,H,W] -> channels-last [D,H,W,24] (one-time / on-change re-layout). */
int sr_lbs_weights_to_channels_last(const float* ws_ncdhw, float* ws_cl, int D, int H, int W,
                                    cudaStream_t s);

/* Composite deformer D(p) = LBS(p + MLPTranslator(p, cond[b])) (model/Deformer.py:15-20).
 *   pts [P,3]; batch_inds [P] int64 or NULL (then b = i / pts_per_frame: "mesh mode");
 *   conds [F,condlen]; lbs == NULL -> translator only.
 *   out d[P,3]; optional offset[P,3] (MLPTranslator.offset), optional jac[P,3,3]
 *   (= d D / d p, row r = gradient of output r: utils/utils.py:106-120), optional
 *   corner_idx[P,3] int32 (LBS trilinear corner indices).                                 */
int sr_deform_forward(const sr_mlp_desc* net, const sr_lbs_params* lbs, const float* pts,
                      const int64_t* batch_inds, int64_t pts_per_frame, const float* conds,
                      int condlen, int64_t P, float* d, float* offset, float* jac,
                      int32_t* corner_idx, cudaStream_t s);

/* Rendering network: cat([p, PE(view), n, feat]) -> rgb in [-1,1] (RenderNet.py:54-89). */
int sr_render_forward(const sr_mlp_desc* net, const float* pts, const float* normals,
                      const float* views, const float* feat, int nfeat, int64_t P, float* rgb,
                      cudaStream_t s);

/* ------------------------------------------------------------------------------------------
 * Surface-point finder ("sphere tracer"), OptimizeSurfacePs (utils/FindSurfacePs.py:114-163).
 * State arrays (device, caller allocated):
 *   pts[P,3] in/out, rays[P,3], batch_inds[P] int64, active_a/active_b [P] int32 work lists,
 *   counters[4] int32, converged[P] bytes (out).
 * sr_trace_init evaluates the initial test and builds the first active list;
 * sr_trace_iter performs ONE damped-Newton iteration on the active list (update + re-test)
 * and writes the next list.  The host launches it `times` times back to back -- no host
 * sync; an empty list makes the launch a no-op.  dnet == NULL means the identity deformer
 * D(p) = p (then lbs must be NULL too).
 * ------------------------------------------------------------------------------------------ */
typedef struct sr_trace_params {
  float cam_pos[3];
  float dthreshold;   /* |f| < dthreshold                       */
  float athreshold;   /* angle (degrees) < athreshold           */
  float w1, w2;       /* loss = w1*|f| + w2*sin(angle)          */
} sr_trace_params;

int sr_trace_step(const sr_mlp_desc* sdf, const sr_mlp_desc* dnet, const sr_lbs_params* lbs,
                  const sr_trace_params* tp, float* pts, const float* rays,
                  const int64_t* batch_inds, const float* conds, int condlen, int64_t P,
                  const int32_t* active_in, int32_t* active_out, int32_t* counters, int iter,
                  uint8_t* converged, cudaStream_t s);

/* Reverse-mode variant of sr_trace_step (same contract, same results up to rounding): the
 * gradient of the scalar loss is obtained with one forward + one backward sweep per network
 * (2 x (F_s+F_d) per ray-iteration instead of the 4 x of forward-mode tangents), which is what
 * the reference's autograd.grad does (FindSurfacePs.py:148).  `scratch` holds act'(z) of the
 * hidden layers between the two sweeps: sr_trace_scratch_bytes() bytes, caller allocated.
 * Requires every layer's `wb`. */
int64_t sr_trace_scratch_bytes(void);
int sr_trace_step_rev(const sr_mlp_desc* sdf, const sr_mlp_desc* dnet, const sr_lbs_params* lbs,
                      const sr_trace_params* tp, float* pts, const float* rays,
                      const int64_t* batch_inds, const float* conds, int condlen, int64_t P,
                      const int32_t* active_in, int32_t* active_out, int32_t* counters, int iter,
                      uint8_t* converged, float* scratch, cudaStream_t s);

/* Geometry part of shading at converged points (infer path, model/network.py:356-361;
 * utils/utils.py:155-169): n = normalize(grad f), cardinal ray = normalize(J^-1 v)
 * (fallback v when |det J|<1e-4), feat = rendcond, d = D(p).                             */
int sr_shade_geometry(const sr_mlp_desc* sdf, const sr_mlp_desc* dnet, const sr_lbs_params* lbs,
                      const float* pts, const float* rays, const int64_t* batch_inds,
                      const float* conds, int condlen, int64_t P, float* normals, float* crays,
                      float* feat, int nfeat, float* dpos, uint8_t* inv_ok, cudaStream_t s);

/* ------------------------------------------------------------------------------------------
 * Tensor-core engine for the dense layers (Hopper wgmma + TMA bulk copies): split-BF16 GEMM
 * (x = b1 + b2, three bf16 MMAs per product, fp32 accumulation in registers), one launch per
 * layer,  C = act(A * W^T + b)  with the epilogue (bias, activation, forward-mode tangent scaling,
 * skip concat, re-split) fused.  Operands are kept in global memory in the canonical no-swizzle
 * tile layout of the wgmma descriptors (see csrc/tc_gemm.cu):
 *   sr_tc_act_bytes(M,K) / sr_tc_weight_bytes(N,K): buffer sizes of tiled activations / weights
 *   sr_tc_pack_rows    : fp32 row-major [M][K] (ld) -> tiled split-bf16 activations
 *   sr_tc_pack_weights : fp32 row-major [N][K] (ld) effective weights -> tiled split-bf16
 *   sr_tc_linear       : one layer. A (tiled, K), W (tiled, N x K), bias [pad256(N)];
 *                        n_valid output columns; ch = rows per point (1, or 4 = value + 3
 *                        tangents: tangent rows get act'(z_value) * acc, no bias);
 *                        A_next (tiled, K_next columns, may be NULL) receives scale*act(.) with
 *                        columns [n_valid, n_valid+skip_n) taken from skip_src (the skip concat of
 *                        network.py:88-89) and the rest zero; out (fp32 [M][out_ld], may be NULL)
 *                        receives result columns [out_col0, out_col0+out_n); dstash (fp32
 *                        [M][pad256(N)], may be NULL) receives act'(z) of value rows; mul_tiles
 *                        (may be NULL) switches the epilogue to the reverse-mode sweep
 *                        out = acc * act'(z_prev): act' is recomputed from the previous layer's
 *                        stored output a = mul_tiles (tiled, mul_K columns, stored as mul_scale*a by
 *                        the forward pass) -- softplus100: 1-exp(-100a), relu: a>0 (mul_act) -- so
 *                        the forward sweep writes no separate stash; m_dev (may be NULL) is a
 *                        device-side row count <= M (active rays).
 * Replaces the nn.Linear / cuBLAS calls of ImplicitNetwork / MLPTranslator / RenderNet for
 * large batches (model/network.py:85-94, Deformer.py:64-69, RenderNet.py:80-88).
 * ------------------------------------------------------------------------------------------ */
/* embedded network input, fp32 [P*ch][ld]: PE(p) (+ cond[b]); tangent rows hold d/dp of it.
 * pe_w is a HOST array of `multires` band weights. */
int sr_tc_embed(const float* pts, int64_t P, int multires, const float* pe_w, int ch,
                const float* conds, const int64_t* batch_inds, int64_t pts_per_frame, int condlen,
                float* out, int ld, const int32_t* index /* optional active list */,
                const int32_t* m_dev /* optional device-side count */, cudaStream_t s);
/* Backward of sr_tc_embed w.r.t. the points: gx [P*ch, ld] -> gp [P,3] (value row: d PE/dp; tangent rows: second
 * derivative of the encoding).  The latent-code columns are a plain slice of gx (value rows). multires <= 8. */
int sr_tc_embed_backward(const float* pts, int64_t P, int multires, const float* pe_w, int ch, const float* gx, int ld,
                         float* gp, cudaStream_t s);
int64_t sr_tc_act_bytes(int64_t M, int K);
int64_t sr_tc_weight_bytes(int N, int K);
int sr_tc_pack_rows(const float* src, int64_t M, int K, int ld, void* dst, const int32_t* m_dev,
                    cudaStream_t s);
int sr_tc_pack_weights(const float* w, int N, int K, int ld, void* dst, cudaStream_t s);
int sr_tc_linear(const void* A, const void* W, const float* bias, int64_t M, int N, int K,
                 int n_valid, int act, int ch, void* A_next, int K_next, float scale,
                 const float* skip_src, int skip_n, int skip_ld, float* out, int out_ld,
                 int out_col0, int out_n, float* dstash, const void* mul_tiles, int mul_K, int mul_act,
                 float mul_scale, const int32_t* m_dev, cudaStream_t s);

/* Mesh rasteriser for the ray seed (replaces pytorch3d.renderer.MeshRasterizer in model/network.py:492 / :345 with
 * faces_per_pixel = 1, blur_radius = 0, perspective_correct = True; consumer: utils/FindSurfacePs.py:5-29).
 * verts_screen [N,V,3] = (pixel x = column, pixel y = row, camera depth z); faces [F,3] int64; keys = scratch of
 * N*H*W uint64.  pix_to_face [N,H,W] int64 (n*F + f, -1 = empty), bary [N,H,W,3], zbuf [N,H,W] or NULL. */
int sr_raster_mesh(const float* verts_screen, const int64_t* faces, int64_t N, int64_t V, int64_t F, int H, int W,
                   uint64_t* keys, int64_t* pix_to_face, float* bary, float* zbuf, cudaStream_t s);

/* Training half of the tensor-core engine (model/network.py:599-639, 774-796: loss.backward() and the parameter
 * VJPs; in a reverse launch (`mul_tiles` != NULL) `dstash` is an INPUT: the fp32 act'(z) the forward launch of the
 * previous layer wrote (leading dimension = that layer's width rounded up to 256), or NULL to recompute act' from the
 * activation tiles.
 * sr_tc_linear with mul_tiles != NULL is the reverse sweep of one layer; with
 * ch == 4 it propagates the cotangents of forward-mode rows (value + 3 tangents per point), i.e. second order.
 *   sr_tc_wgrad   dW[N x K] (row-major, ld) = delta^T x over M rows; delta / x = tiled split-bf16 activations with
 *                 Kd / Kx feature columns (each a multiple of 32); `part` = scratch of
 *                 sr_tc_wgrad_partial_bytes(M, Kd, Kx, NULL) bytes.  wgmma with MN-major operands: no transposes.
 *   sr_tc_colsum  partial[slice][k] = sum over rows with row % ch == 0 (value rows) of the tiled activations: the
 *                 bias gradient after a sum over slices.
 *   sr_tc_unpack_rows   tiled split-bf16 -> fp32 [M][K] (inverse of sr_tc_pack_rows).                           */
int64_t sr_tc_wgrad_partial_bytes(int64_t M, int Kd, int Kx, int* splits_out);
void sr_tc_debug_wgrad_desc_swap(int v);   /* test knob: 1 swaps the LBO / SBO descriptor fields */
int sr_tc_wgrad(const void* D, int Kd, const void* X, int Kx, int64_t M, float* part, float* dW, int N, int K,
                int ld, cudaStream_t s);
int sr_tc_colsum(const void* T, int64_t M, int K, int ch, float* partial, int slices, cudaStream_t s);
int sr_tc_unpack_rows(const void* T, int64_t M, int K, int Kpad, float* out, int ld, cudaStream_t s);

/* Whole-sweep entry points: all launches of one forward / backward evaluation of an MLP from ONE call (per-layer
 * operands = the module's persistent packs).  forward: x0 [M, ld] fp32 rows (ld a multiple of 32, the first d_in
 * columns = the embedded input) -> out [M, n_out] (n_out = 0: all n_last columns); a skip layer's input is
 * cat(previous output, x0[:, :d_in]) / sqrt(2).  Keeps the input tiles (A_in), every hidden layer's activation tiles
 * (acts[i], sr_tc_act_bytes(M, k_{i+1})) and, for softplus layers, the fp32 act'(z) (stashes[i] [M, pad256(n_i)] or
 * NULL).  m_dev (may be NULL): device-side row count <= M (active rays).  backward: gout [M, n_last] -> dW[l] [n,k] / db[l] [n] (NULL entries are
 * skipped) and x0_grad [M, ld] (or NULL); D0 / D1 = two delta tile buffers of sr_tc_act_bytes(M, widest layer),
 * part = sr_tc_wgrad_partial_bytes scratch for the widest pair, colsum_ws = colsum_slices x widest floats,
 * g_skip [M, g_skip_ld] scratch when a layer has a skip connection. */
typedef struct sr_tc_layer {
  const void* W;          /* packed weights, forward orientation (sr_tc_pack_weights of [n,k]) */
  const void* Wb;         /* packed W^T ([k,n]) for the reverse launch */
  const float* bias;      /* padded to a multiple of 256 */
  const float* zero_bias; /* zeros, pad256(k) */
  int n, k, act, skip;
} sr_tc_layer;
int sr_tc_mlp_forward(const sr_tc_layer* layers, int L, const float* x0, int64_t M, int ld, int d_in, int ch, void* A_in,
                      void* const* acts, float* const* stashes, float* out, const int32_t* m_dev, int n_out,
                      cudaStream_t s);
int sr_tc_mlp_backward(const sr_tc_layer* layers, int L, int64_t M, int ld, int d_in, int ch, const float* gout,
                       const void* A_in, void* const* acts, float* const* stashes, void* D0, void* D1, float* part,
                       float* colsum_ws, int colsum_slices, float* const* dW, float* const* db, float* x0_grad,
                       float* g_skip, int g_skip_ld, cudaStream_t s);

/* Batched 3x3 singular values (descending) + right singular vectors (columns of V, may be NULL), and the
 * backward of a function of the VALUES: gJ = sum_i gS_i u_i v_i^T.  Replaces `torch.svd(Jacobs.cpu())` of the
 * def_regu block (model/network.py:573-575).  J, V, gJ: [n,3,3] row-major; S, gS: [n,3]. */
int sr_svals3x3_f32(const float* J, float* S, float* V, int64_t n, cudaStream_t s);
int sr_svals3x3_bwd_f32(const float* J, const float* S, const float* V, const float* gS, float* gJ, int64_t n,
                        cudaStream_t s);

/* Weight-normalised layers (torch.nn.utils.weight_norm, dim 0; model/network.py:60-61, model/RenderNet.py): the
 * effective weights w = g v / ||v|| of up to 12 layers in one launch, and the backward of that map
 * (gv, gg from gw; gw may be NULL = no gradient reached this layer, gw_ld = row stride of gw in floats).
 * inv_norm [n] is written by the forward call and read by the backward call. */
typedef struct sr_wn_layer {
  const float* v;       /* [n][k] direction parameter (weight_v) */
  const float* g;       /* [n] magnitude parameter (weight_g) */
  float* w;             /* [n][k] effective weight (forward out) */
  float* inv_norm;      /* [n] 1 / ||v|| (forward out, backward in) */
  const float* gw;      /* [n][gw_ld] gradient of w (backward in) or NULL */
  float* gv;            /* [n][k] (backward out) */
  float* gg;            /* [n] (backward out) */
  int32_t n, k, gw_ld, pad_;
} sr_wn_layer;
int sr_weight_norm_forward(const sr_wn_layer* layers, int L, cudaStream_t s);
int sr_weight_norm_backward(const sr_wn_layer* layers, int L, cudaStream_t s);

/* Borderline decisions.  The tensor-core engine's values carry up to ~2.4e-5 of absolute error, so
 * a sign (`> balance`, MCAcc/seg3d_lossless.py:333-346) or threshold (`< dthreshold`,
 * utils/FindSurfacePs.py:120-127) decision on a value inside that band is re-taken on the fp32 FFMA engine:
 * sr_band_select lists the ids with |v - center| < eps (device-side count, caller zeroes it),
 * sr_sdf_forward_indexed re-evaluates exactly those points and overwrites sdf[id].  For the tracer,
 * sr_tc_trace_mid (below) lists the rays whose convergence test could flip within (eps_f, eps_a [degrees]) and
 * sr_trace_step_rev (test-only: active_out = NULL, active_in = that list) decides them. */
int sr_band_select(const float* values, int64_t n, float center, float eps, int32_t* list,
                   int32_t* counter, cudaStream_t s);
int sr_sdf_forward_indexed(const sr_mlp_desc* net, const float* pts, int64_t P, const int32_t* index,
                           const int32_t* m_dev, float* sdf, cudaStream_t s);
/* Same contract for the first `cap` entries of the list, as one column-split launch per layer (fp32 FMAs): short lists
 * do not pay the persistent engine's per-tile latency.  work = sr_sdf_small_work_bytes(cap) bytes. */
int64_t sr_sdf_small_work_bytes(int cap);
int sr_sdf_forward_small(const sr_mlp_desc* net, const float* pts, int64_t P, const int32_t* index,
                         const int32_t* m_dev, float* sdf, void* work, int cap, cudaStream_t s);

/* Pointwise stages of the tensor-core tracer (one OptimizeSurfacePs iteration =
 * embed -> sr_tc_mlp_forward (activations kept per layer) -> sr_tc_trace_mid -> sr_tc_linear x
 * layers (reverse sweep, mul_tiles = the forward activations) -> sr_tc_trace_update).  All take an optional active
 * list + device-side count so the host never synchronises.  pw_s / pw_d are HOST arrays. */
int sr_tc_trace_mid(const int32_t* index, const int32_t* m_dev, int64_t P, const float* pts,
                    const float* rays, const int64_t* batch_inds, const float* f, const float* off,
                    const sr_lbs_params* lbs, const sr_trace_params* tp, int do_update,
                    uint8_t* converged, float* dsdf, float* ddef, int ld, float* aux,
                    int32_t* recheck /* [P] or NULL */, int32_t* recheck_count, float eps_f, float eps_a,
                    cudaStream_t s);
int sr_tc_trace_update(const int32_t* index, const int32_t* m_dev, int64_t P, float* pts,
                       const float* gs, int gs_ld, const float* gskip, int gk_ld, const float* gd,
                       int gd_ld, const float* aux, int mr_s, const float* pw_s, int mr_d,
                       const float* pw_d, int32_t* active_out, int32_t* counter_out,
                       const uint8_t* converged /* or NULL */, cudaStream_t s);

/* Shading on the tensor-core engine: sr_tc_shade_point turns the 4-rows-per-point outputs of the
 * SDF (value / grad f in column 0) and translator (offset / d offset) sweeps into normals,
 * cardinal rays (J^-1 v, fallback v when |det J| < 1e-4) and D(p); sr_tc_render_embed builds
 * cat([p, PE(view), n, feat]) rows for the rendering network (RenderNet.py:73-74); feat is read
 * from row p*feat_row_stride of a [*, feat_ld] matrix starting at column feat_col0. */
int sr_tc_shade_point(int64_t P, const float* pts, const float* rays, const int64_t* batch_inds,
                      const float* sdf4, int ld_s, const float* off4, const sr_lbs_params* lbs,
                      float* normals, float* crays, float* dpos, uint8_t* inv_ok, cudaStream_t s);
int sr_tc_render_embed(int64_t P, const float* pts, const float* views, const float* normals,
                       const float* feat, int feat_ld, int feat_col0, int nfeat, int feat_row_stride,
                       int multires, const float* pw, float* out, int ld, cudaStream_t s);

/* ------------------------------------------------------------------------------------------
 * Coarse-to-fine SDF grid plumbing (Seg3dLossless, MCAcc/seg3d_lossless.py:266-372).
 *   cand[z,y,x] = any(flag over the zero-padded 3x3x3 neighbourhood)
 *                 && !calculated[z*sz, y*sy, x*sx]
 *   flag/cand: [D,H,W] bytes (level lattice); calculated: [fD,fH,fW] bytes (final grid).
 * Replaces the fp32 conv3d dilation (:296), the coords_accum masking (:299-301) and the
 * 27-neighbour gathering of the conflict loop (:354-372).
 * ------------------------------------------------------------------------------------------ */
int sr_seg3d_candidates(const uint8_t* flag, const uint8_t* calculated, uint8_t* cand, int D,
                        int H, int W, int sz, int sy, int sx, int fD, int fH, int fW,
                        cudaStream_t s);
/* Per-pass glue around the query function (seg3d_lossless.py:94-101, 318-346):
 *   gather : lin[n] (linear ids on the [D,H,W] level lattice) -> world points [n,3] with
 *            batch_eval's arithmetic (c/res + (1/res)/2) * (bmax-bmin) + bmin, one rounding per
 *            op; interp[n] = grid[lin]; calculated[final-grid voxel] = 1.  bmin/bmax: HOST [3].
 *   scatter: grid[lin] = values; conflict[lin] = (interp-balance)*(values-balance) < 0 on a
 *            zeroed level-sized byte mask; *n_conflicts = how many (device int32). */
int sr_seg3d_gather(const int64_t* lin, int64_t n, int H, int W, int sz, int sy, int sx, int fD,
                    int fH, int fW, const float* bmin, const float* bmax, const float* grid,
                    float* points, float* interp, uint8_t* calculated, cudaStream_t s);
int sr_seg3d_scatter(const int64_t* lin, int64_t n, const float* values, const float* interp,
                     float balance, float* grid, uint8_t* conflict, int64_t conflict_bytes,
                     int32_t* n_conflicts, cudaStream_t s);

#ifdef __cplusplus
}
#endif
#endif /* SELFRECON_B200_H_ */
