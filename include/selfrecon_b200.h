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
 *   With C == 0 the C-sized arrays (input, output, grad_output, grad_input, gg_input,
 *   grad_grad_output) may be NULL; corner_idx and grad_grid (zeros) are still written.
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
 *   sr_tc_pack_weights : fp32 row-major [N][K] (ld) effective weights -> tiled split-bf16 (64-column
 *                        tiles when N <= 64, else 256: a pack is only valid for launches of the same N)
 *   sr_tc_linear       : one layer. A (tiled, K), W (tiled, N x K), bias [pad256(N)];
 *                        n_valid output columns; ch = rows per point (1, or 4 = value + 3
 *                        tangents: tangent rows get act'(z_value) * acc, no bias);
 *                        A_next (tiled, K_next columns, may be NULL) receives scale*act(.) with
 *                        columns [n_valid, n_valid+skip_n) taken from skip_src (the skip concat of
 *                        network.py:88-89) and the rest zero (K_next may exceed pad256(N): the
 *                        chunks past it hold only skip / zero columns and are written by a second,
 *                        small launch after the layer kernel); out (fp32 [M][out_ld], may be NULL)
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
 * derivative of the encoding).  The latent-code columns are a plain slice of gx (value rows). multires <= 8.
 * gk [P, gk_ld] (ch = 1 only, or NULL) is added to gx's encoding columns: a skip layer's part of a reverse sweep. */
int sr_tc_embed_backward(const float* pts, int64_t P, int multires, const float* pe_w, int ch, const float* gx, int ld,
                         const float* gk, int gk_ld, float* gp, cudaStream_t s);
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

/* Shaded images of OptimNetwork.infer (model/network.py:318-338 with infer.py:90's HardPhongShader), forward only.
 * sr_mesh_vertex_normals: pytorch3d's Meshes.verts_normals_packed for N frames of world vertices [N,V,3] sharing one
 *   face table [F,3]: the sum of the unnormalised face normals (v2-v1) x (v0-v1) over the incident faces, divided by
 *   max(|sum|, 1e-6).  vf_offsets [V+1] / vf_faces = CSR of each vertex's incident faces in ascending order; the sum
 *   follows that order (no atomics: bit-identical reruns).  normals [N,V,3].
 * sr_shade_phong: pytorch3d's phong_shading + hard_rgb_blend with faces_per_pixel = 1, one point light and one
 *   material, on the fragments sr_raster_mesh writes (pix_to_face [N,H,W] = n*F + f or -1, bary [N,H,W,3]).
 *   verts / normals / colors [N,V,3] (colors NULL = white), cam_pos / light_pos [N,3] device arrays (per image frame).
 *   out [N,H,W,4] (16-byte aligned): (rgb, 1) on covered pixels, (background, 0) elsewhere. */
typedef struct sr_phong_params {
  float light_ambient[3], light_diffuse[3], light_specular[3];
  float mat_ambient[3], mat_diffuse[3], mat_specular[3];
  float shininess;
  float background[3];
} sr_phong_params;
int sr_mesh_vertex_normals(const float* verts, const int64_t* faces, const int64_t* vf_offsets, const int64_t* vf_faces,
                           int64_t N, int64_t V, int64_t F, float* normals, cudaStream_t s);
int sr_shade_phong(const float* verts, const float* normals, const float* colors, const int64_t* faces, int64_t N,
                   int64_t V, int64_t F, const int64_t* pix_to_face, const float* bary, int H, int W,
                   const float* cam_pos, const float* light_pos, const sr_phong_params* params, float* out,
                   cudaStream_t s);

/* Soft point-cloud silhouette of the template (model/network.py:495-505: pytorch3d 0.4.0 PointsRasterizer with
 * points_per_pixel = K and radius r in NDC, then AlphaCompositor(background_color=None), all features 1), forward and
 * backward.  pts_screen [N,V,3] = (col, row, view-space Z) per frame, pixel centres at integers.  Point p covers pixel
 * (i, j) iff Z >= 0 and d2 = (2/W)^2 (col-j)^2 + (2/H)^2 (row-i)^2 < r^2; each pixel keeps its K covering points of
 * smallest (Z, index) and composites w = 1 - d2/r^2: mask = 1 - prod (1 - w).  Pixels are SR_POINTS_TILE square tiles.
 *   sr_points_silhouette_list_capacity: slots of the tile lists (N * V * tiles per point), SR_EINVAL if invalid.
 *   sr_points_silhouette_bin: order [N,V] = each frame's point indices in (Z, index) order (a stable sort by Z);
 *     writes per (frame, rank) a fixed number of slots: tile_keys = n * tiles + tile, tile_points = the point index;
 *     unused slots hold key N * tiles and point -1.  A stable sort of the keys (carrying tile_points) then gives
 *     every tile's points in (Z, index) order; tile_offsets [N * tiles + 1] delimit them.
 *   sr_points_silhouette_forward: mask [N,H,W] plus the backward's per-pixel state: kth_key = (Z bits << 32 | index)
 *     of the K-th kept point (all ones when fewer than K cover), prod = product of the nonzero (1 - w), zeros = count
 *     of w == 1.
 *   sr_points_silhouette_backward: grad_pts [N,V,3] = dL/d(col, row, Z) (Z gets 0) for grad_mask [N,H,W].
 *     No atomics: bit-identical reruns. */
#define SR_POINTS_TILE 16
int64_t sr_points_silhouette_list_capacity(int64_t N, int64_t V, int H, int W, float radius);
int sr_points_silhouette_bin(const float* pts_screen, const int64_t* order, int64_t N, int64_t V, int H, int W,
                             float radius, int64_t* tile_keys, int32_t* tile_points, cudaStream_t s);
int sr_points_silhouette_forward(const float* pts_screen, const int64_t* tile_offsets, const int32_t* tile_points,
                                 int64_t N, int64_t V, int H, int W, float radius, int K, float* mask,
                                 uint64_t* kth_key, float* prod, int32_t* zeros, cudaStream_t s);
int sr_points_silhouette_backward(const float* pts_screen, const float* grad_mask, const uint64_t* kth_key,
                                  const float* prod, const int32_t* zeros, int64_t N, int64_t V, int H, int W,
                                  float radius, float* grad_pts, cudaStream_t s);

/* Template mesh regularisers of OptimNetwork.computeTmpPcLoss (model/network.py:655-670): pytorch3d 0.4.0's
 * mesh_laplacian_smoothing(method='uniform'), mesh_edge_loss(target_length=0.) and mesh_normal_consistency of one mesh,
 * verts [V,3] float, faces [F,3] int64, V <= 2^31.
 * Topology, once per face table (Meshes._compute_packed):
 *   sr_mesh_reg_edge_keys: keys [3F]; entry 3f+k = the edge opposite corner k of face f as the hash V*min + max of its
 *     two vertex ids, or -1 when either id is outside [0, V).  The caller sorts the keys stably (keeping perm).
 *   sr_mesh_reg_edge_runs: over the n sorted keys: head[i] = 1 where a run of equal keys (one unique edge) starts, else
 *     0; npairs[i] = the run's pair count at a head ((m-1)^2 - (m-2) for a run of m >= 2 entries), else 0.
 *   sr_mesh_reg_topology: head_cum / pair_cum = inclusive prefix sums of head / npairs, E = head_cum[3F-1],
 *     P = pair_cum[3F-1].  Writes edges [E,2] (a <= b, ascending hash), face_to_edge [F,3], dir_keys [2E] (V*a+b and
 *     V*b+a of each edge: sorted by the caller into the directed neighbour CSR) and pairs [P,4] = (a, b, o_i, o_j), the
 *     opposite corners of pytorch3d's literal list [e[i], e[j]] for i in range(m-1) for j in range(1, m) if i != j over
 *     each edge's entries e in ascending (face, corner) order.
 * sr_mesh_reg_forward: out [3] = (sum_i |(L v)_i| / V, sum_e |v_a - v_b|^2 / E, sum_p (1 - cos(n_i, -n_j)) / P or 0),
 *   fp64 inside.  nbr_off [V+1] / nbr = each vertex's directed neighbours (a self-edge twice), ascending; L v =
 *   mean of the neighbours - v (-v without neighbours).  n = (v_b - v_a) x (v_o - v_a), exactly 0 with no gradient
 *   when o = a, o = b or a = b; cos = w12 / sqrt(max(w1 w2, 1e-16)).  Workspace for the backward: u [V,3] = (L v)_i / |(L v)_i| (0 at a zero norm), dn [P,6] = d(1 - cos)/dn_i,
 *   d/dn_j; partials = 3 * SR_MESH_REG_BLOCKS doubles.  Two launches: block partials, then a fixed-order sum.
 * sr_mesh_reg_backward: grad_verts [V,3] for the cotangent grad_out [3] (device), one thread per vertex gathering over
 *   its neighbours and its (pair, role) entries vp_off [V+1] / vp_ent (= 4 p + role, role = the vertex's column of
 *   pairs), in CSR order.
 * pairs, dn and vp_ent may be NULL when P = 0.  No atomics: bit-identical reruns. */
#define SR_MESH_REG_BLOCKS 528
int sr_mesh_reg_edge_keys(const int64_t* faces, int64_t F, int64_t V, int64_t* keys, cudaStream_t s);
int sr_mesh_reg_edge_runs(const int64_t* sorted_keys, int64_t n, int64_t* head, int64_t* npairs, cudaStream_t s);
int sr_mesh_reg_topology(const int64_t* faces, const int64_t* sorted_keys, const int64_t* perm, const int64_t* head_cum,
                         const int64_t* pair_cum, int64_t F, int64_t V, int64_t E, int64_t P, int64_t* edges,
                         int64_t* face_to_edge, int64_t* dir_keys, int64_t* pairs, cudaStream_t s);
int sr_mesh_reg_forward(const float* verts, int64_t V, int64_t E, int64_t P, const int64_t* edges,
                        const int64_t* nbr_off, const int64_t* nbr, const int64_t* pairs, double* u, double* dn,
                        double* partials, float* out, cudaStream_t s);
int sr_mesh_reg_backward(const float* verts, int64_t V, int64_t E, int64_t P, const int64_t* nbr_off,
                         const int64_t* nbr, const int64_t* pairs, const int64_t* vp_off, const int64_t* vp_ent,
                         const double* u, const double* dn, const float* grad_out, float* grad_verts, cudaStream_t s);

/* Texture atlas of the reconstruction (texture_mesh_extract.py:57-144: VideoAvatar's Isomapper aggregation), over the
 * T atlas texels a UV face covers (the UV raster: sr_raster_mesh on the atlas), S <= SR_TEXTURE_MAX_SLOTS slots each.
 * Slots are slot-major: slot_rgb [S][3][T] (colour in [0,1], planar), slot_alpha [S][T] (c0 = cos(max_angle) when
 * empty), slot_view [S][T] (frame id, -1 when empty); min_alpha / min_slot [T] = the smallest slot alpha and the first
 * slot holding it (start: c0, 0).
 *   sr_texture_accumulate: one frame.  texel_face [T] (face of F), texel_bary [T,3]; verts_screen [V,3] = the frame's
 *     (col, row, Z), pixel centres at integers; vert_weight [V] = max(0, -n_v . d_v); face_usable [F] (0/1); image
 *     [H,W,3] uint8 in its own channel order.  alpha = sum b_i w_i over a usable face (0 otherwise); when alpha >
 *     min_alpha the slot min_slot takes (bilinear(image, sum b_i s_i) / 255 with clamp-to-edge, alpha, frame_id >= 0)
 *     and the pair is rescanned.
 *   sr_texture_finish: count = #slots with alpha > c0, mask_final = count >= min_views, view_id = frame of the first slot
 *     with the largest alpha (-1 unless mask_final), tex_median = per-channel median of the filled slots (mean of the two
 *     middle values for an even count; 0 unless mask_final).  Written at texel_index [T] of the outputs tex_median
 *     [R*R,3], mask_final / view_id / count [R*R]; other texels are left as they are.
 * One thread owns each texel (no atomics: bit-identical reruns). */
#define SR_TEXTURE_MAX_SLOTS 64
int sr_texture_accumulate(int64_t T, int S, const int32_t* texel_face, const float* texel_bary,
                          const float* verts_screen, const int64_t* faces, int64_t V, int64_t F, const float* vert_weight,
                          const uint8_t* face_usable, const uint8_t* image, int H, int W, int frame_id,
                          float* slot_rgb, float* slot_alpha, int32_t* slot_view, float* min_alpha, int32_t* min_slot,
                          cudaStream_t s);
int sr_texture_finish(int64_t T, int S, const int64_t* texel_index, const float* slot_rgb, const float* slot_alpha,
                      const int32_t* slot_view, float c0, int min_views, float* tex_median, uint8_t* mask_final,
                      int32_t* view_id, int32_t* count, cudaStream_t s);

/* Skin-weight volume of a new sequence (model/Deformer.py:235-284, utils/LBSWsmpl.py:2-52: compute_lbswField and
 * smooth_weights).  Volumes are [C][D][H][W] float (x fastest), (W, H, D) = the resolutions; bmin / bmax are HOST [3].
 *   sr_lbsw_knn_blend: verts [V,3], vert_ws [V,C].  Voxel (i, j, l) has the centre u * (hi - lo) + lo with
 *     u = i / W + (1 / W) / 2 (i / (W - 1) with align_corners), every fp32 operation rounded on its own (no FMA).  Its
 *     k nearest vertices by exact fp32 differences, ordered by (d^2, index), are blended with w_n = 1 / min(max(d_n,
 *     1e-4), 1) normalised by their sum: field[c] = sum_n w_n vert_ws[idx_n, c] in ascending distance order.
 *     centres [W*H*D,3] (may be NULL) receives the voxel centres.  1 <= k <= min(V, SR_LBSW_MAX_K),
 *     1 <= C <= SR_LBSW_MAX_C.
 *   sr_lbsw_smooth_pass: one Jacobi pass src -> dst (distinct buffers): interior voxels become (c - mean) * 0.7 + mean,
 *     mean = the six neighbours of src in the order (+z, -z, +y, -y, +x, -x) / 6; boundary voxels keep theirs; every
 *     voxel is divided by its channel sum; with cut > 0, values below cut become 0.
 *   sr_lbsw_cut: field[t] < cut -> 0 in place over n values (the utils.LBSWsmpl variant with no smoothing pass).
 * No atomics: bit-identical reruns. */
#define SR_LBSW_MAX_K 32
#define SR_LBSW_MAX_C 32
int sr_lbsw_knn_blend(const float* verts, const float* vert_ws, int V, int C, const float* bmin, const float* bmax,
                      int W, int H, int D, int align_corners, int k, float* field, float* centres, cudaStream_t s);
int sr_lbsw_smooth_pass(const float* src, float* dst, int C, int D, int H, int W, float cut, cudaStream_t s);
int sr_lbsw_cut(float* field, int64_t n, float cut, cudaStream_t s);

/* Device-resident frames of a sequence (dataset/dataset.py:89-102: SceneDataset.__getitem__ decoded once).  Store:
 * img_store / normal_store uint8 [F,H,W,3] in file (BGR) order as cv2 reads it; mask_store uint32 [F,H,ceil(W/32)],
 * bit (c & 31) of word (c >> 5) = column c has a nonzero channel, rows padded to whole words.  For n < N and
 * f = frame_ids[n] (device int64, 0 <= f < F, checked by the caller: rows with other ids are left unwritten):
 *   img [N,H,W,3]    = (x / 255 - 0.5) * 2                 in file order
 *   mask [N,H,W]     = 1 where the bit is set, else 0
 *   normal [N,H,W,3] = 2 x / 255 - 1                       channels reversed (RGB)
 * each fp32 operation rounded on its own, so the results are bit-identical to the numpy expressions.  Any output may be
 * NULL; the store plane an output reads must not be.  SR_EINVAL for F, H or W <= 0, N < 0 or a missing plane. */
int sr_frames_decode(const uint8_t* img_store, const uint32_t* mask_store, const uint8_t* normal_store, int F, int H,
                     int W, const int64_t* frame_ids, int64_t N, float* img, float* mask, float* normal,
                     cudaStream_t s);

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
 * NULL).  m_dev (may be NULL): device-side row count <= M (active rays).  backward: the one reverse sweep, from
 * gout [M, gout_ld] (gout_ld >= n_last; its first n_last columns are the cotangent) -> dW[l] [n,k] / db[l] [n] (dW / db
 * may be NULL arrays, NULL entries are skipped) and x0_grad [M, ld] (or NULL); D0 / D1 = two delta tile buffers of
 * sr_tc_act_bytes(M, widest layer); only when some dW[l] / db[l] is requested: A_in = the forward's input tiles,
 * part = sr_tc_wgrad_partial_bytes scratch, the largest over the layers' (Kd, Kx) pairs, colsum_ws = colsum_slices x
 * widest floats.  g_skip [M, g_skip_ld] receives the skip layer's part of the input gradient (its first d_in columns)
 * when a layer has a skip connection; more than one skip layer returns SR_EUNSUPPORTED.  The input layer's launch writes
 * the first n_keep columns of x0_grad: Wb_head = NULL takes layers[0].Wb with n_keep = layers[0].k, otherwise Wb_head =
 * sr_tc_pack_weights of the first n_keep rows of W^T (a narrow launch when n_keep <= 64).  fold_skip = 1 then zeroes
 * columns [n_keep, ld) of x0_grad and adds g_skip into its first d_in columns; fold_skip = 0 leaves the skip part in
 * g_skip (sr_tc_embed_backward and sr_tc_trace_update take it as an input) and launches nothing after that layer.
 * m_dev (may be NULL) is passed to the pack and every layer launch; it requires no dW / db and fold_skip = 0. */
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
                       int gout_ld, const void* A_in, void* const* acts, float* const* stashes, void* D0, void* D1,
                       float* part, float* colsum_ws, int colsum_slices, float* const* dW, float* const* db,
                       float* x0_grad, float* g_skip, int g_skip_ld, const void* Wb_head, int n_keep, int fold_skip,
                       const int32_t* m_dev, cudaStream_t s);

/* Batched 3x3 singular values (descending) + right singular vectors (columns of V, may be NULL), and the
 * backward of a function of the VALUES: gJ = sum_i gS_i u_i v_i^T.  Replaces `torch.svd(Jacobs.cpu())` of the
 * def_regu block (model/network.py:573-575).  J, V, gJ: [n,3,3] row-major; S, gS: [n,3]. */
int sr_svals3x3_f32(const float* J, float* S, float* V, int64_t n, cudaStream_t s);
int sr_svals3x3_bwd_f32(const float* J, const float* S, const float* V, const float* gS, float* gJ, int64_t n,
                        cudaStream_t s);

/* Borderline decisions.  The tensor-core engine's values carry up to ~2.4e-5 of absolute error, so
 * a sign (`> balance`, MCAcc/seg3d_lossless.py:333-346) or threshold (`< dthreshold`,
 * utils/FindSurfacePs.py:120-127) decision on a value inside that band is re-taken on the fp32 FFMA engine:
 * sr_band_select lists the ids with |v - center| < eps (device-side count, caller zeroes it),
 * sr_sdf_forward_indexed re-evaluates exactly those points and overwrites sdf[id]. */
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
 * embed -> sr_tc_mlp_forward (activations kept per layer) -> sr_tc_trace_mid -> sr_tc_mlp_backward
 * (reverse sweep over the forward activations, fold_skip = 0) -> sr_tc_trace_update).  All take an optional active
 * list + device-side count so the host never synchronises.  pw_s / pw_d are HOST arrays. */
int sr_tc_trace_mid(const int32_t* index, const int32_t* m_dev, int64_t P, const float* pts,
                    const float* rays, const int64_t* batch_inds, const float* f, const float* off,
                    const sr_lbs_params* lbs, const sr_trace_params* tp, int do_update,
                    uint8_t* converged, float* dsdf, float* ddef, int ld, float* aux, cudaStream_t s);
int sr_tc_trace_update(const int32_t* index, const int32_t* m_dev, int64_t P, float* pts,
                       const float* gs, int gs_ld, const float* gskip, int gk_ld, const float* gd,
                       int gd_ld, const float* aux, int mr_s, const float* pw_s, int mr_d,
                       const float* pw_d, int32_t* active_out, int32_t* counter_out, cudaStream_t s);

/* Shading on the tensor-core engine: sr_tc_shade_point turns grad f [P,3] (the SDF's reverse sweep
 * through sr_tc_embed_backward) and the 4-rows-per-point translator outputs (offset / d offset) into
 * normals, cardinal rays (J^-1 v, fallback v when |det J| < 1e-4) and D(p); sr_tc_render_embed builds
 * cat([p, PE(view), n, feat]) rows for the rendering network (RenderNet.py:73-74); feat is read
 * from row p*feat_row_stride of a [*, feat_ld] matrix starting at column feat_col0. */
int sr_tc_shade_point(int64_t P, const float* pts, const float* rays, const int64_t* batch_inds,
                      const float* grad, const float* off4, const sr_lbs_params* lbs,
                      float* normals, float* crays, float* dpos, uint8_t* inv_ok, cudaStream_t s);
/* sr_tc_shade_point_deformed: sr_tc_shade_point's outputs, bit-identical, plus the deformed-surface normal
 * defnormals [P,3] = normalize(J^-T g) from the same g = grad f (unnormalised) and J = M (I + d offset / dp);
 * where |det J| < 1e-4 it is normalize(J g), the reference's fallback (utils/utils.py:139-152).  cam_R0 (HOST
 * [9], row-major, or null) turns it into the debug image's normal diag(-1,1,-1) R0^T n; the reference rotates
 * every frame of a batch by cameras.R[0] (model/network.py:424), and so does this one. */
int sr_tc_shade_point_deformed(int64_t P, const float* pts, const float* rays, const int64_t* batch_inds,
                               const float* grad, const float* off4, const sr_lbs_params* lbs,
                               float* normals, float* crays, float* dpos, uint8_t* inv_ok, float* defnormals,
                               const float* cam_R0, cudaStream_t s);
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

/* ------------------------------------------------------------------------------------------
 * Front-normal network of the normal-map step (generate_normals.py:116-166; csrc/normal_net.cu).  Activations are
 * fp32 channels-last [B,H,W,C]; a convolution is sr_conv_pack + sr_tc_linear over row chunks.
 *   sr_conv_pack: rows [row0, row0+rows) of the implicit im2col matrix of a kh x kw convolution, column
 *       k = (ky*kw + kx)*Cin + ci, row m = (b*Ho + oy)*Wo + ox, into the tiled split-bf16 layout of
 *       sr_tc_pack_rows (sr_tc_act_bytes(rows, kh*kw*Cin) bytes; tile rows past `rows` are zero).  Zero or
 *       reflection (reflect = 1, pad < H, W) padding, stride 1 or 2; transposed = 1 is ConvTranspose2d in gather
 *       form: input (oy + pad - ky) / stride when that divides exactly and lies in range, else zero.
 *   sr_instance_norm_stats: mean and 1/sqrt(biased var + 1e-5) [B][C] of y [B][HW][C]; float64 partial sums over
 *       fixed 512-pixel slices (scratch: sr_instance_norm_partial_bytes), added in a fixed order: deterministic, and
 *       a sample's result does not depend on B.
 *   sr_instance_norm_apply: out = relu?((y - mean) * rstd) (+ residual), all [B][HW][C]; out may alias y or residual.
 *   sr_normal_unwarp: net output [B,S,S,3] sampled back onto B frames of H x W through the crop boxes [B,4]
 *       (x, y, w, h as floats) as grid_sample(bilinear, zeros, align_corners=True) with x' = 2(c - x)/w - 1, then
 *       generate_normals.py:155-165: |n| < 1e-4 or background -> 0, else (n*0.5 + 0.5)[::-1]*255 truncated:
 *       uint8 BGR [B,H,W,3].  fg (uint8 [B,H,W], nonzero = foreground) may be NULL (no mask).
 * ------------------------------------------------------------------------------------------ */
int sr_conv_pack(const float* x, int B, int H, int W, int Cin, int kh, int kw, int stride, int pad, int reflect,
                 int transposed, int Ho, int Wo, int64_t row0, int64_t rows, void* dst, cudaStream_t s);
int64_t sr_instance_norm_partial_bytes(int B, int64_t HW, int C);
int sr_instance_norm_stats(const float* y, int B, int64_t HW, int C, void* partial, float* mean, float* rstd,
                           cudaStream_t s);
int sr_instance_norm_apply(const float* y, int B, int64_t HW, int C, const float* mean, const float* rstd,
                           const float* residual, int relu, float* out, cudaStream_t s);
int sr_normal_unwarp(const float* net, int B, int S, const float* boxes, const uint8_t* fg, int H, int W,
                     uint8_t* out, cudaStream_t s);

#ifdef __cplusplus
}
#endif
#endif /* SELFRECON_B200_H_ */
