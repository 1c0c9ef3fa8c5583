"""Math helpers of the hot path (reference: utils/utils.py:8-172, 237-316).

Only what the per-frame optimisation step touches is mirrored here; the mesh / texture /
checkpoint-format helpers of the reference are plain torch and out of scope (SURVEY.md 2.1)."""
import numpy as np
import torch
from torch.autograd import Function

from FastMinv import Fast3x3Minv, Fast3x3Minv_backward
from selfreconcode_b200 import ops


class FastDiff3x3MinvFunction(Function):
    @staticmethod
    def forward(ctx, input):
        invs, check = Fast3x3Minv(input.contiguous())
        ctx.save_for_backward(invs, check)
        ctx.mark_non_differentiable(check)
        return invs, check

    @staticmethod
    def backward(ctx, grad_input, grad_check):
        invs, check = ctx.saved_tensors
        return Fast3x3Minv_backward(grad_input.contiguous(), invs), None


class SingularValues3x3Function(Function):
    """Singular values of [P,3,3] matrices on the device (csrc/svals3x3.cu) with the first-order backward
    a spectral loss needs; stands in for `torch.svd(J.cpu())[1]` (model/network.py:573-575)."""

    @staticmethod
    def forward(ctx, J):
        Jc = J.detach().contiguous().float().view(-1, 3, 3)
        S, V = ops.svals3x3(Jc, want_v=True)
        ctx.save_for_backward(Jc, S, V)
        ctx.shape = J.shape
        return S

    @staticmethod
    def backward(ctx, gS):
        Jc, S, V = ctx.saved_tensors
        return ops.svals3x3_backward(Jc, S, V, gS).view(ctx.shape)


def singular_values_3x3(J):
    return SingularValues3x3Function.apply(J)


def quat2mat(quat):
    q = quat / quat.norm(p=2, dim=1, keepdim=True)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    w2, x2, y2, z2 = w.pow(2), x.pow(2), y.pow(2), z.pow(2)
    wx, wy, wz, xy, xz, yz = w * x, w * y, w * z, x * y, x * z, y * z
    return torch.stack([w2 + x2 - y2 - z2, 2 * xy - 2 * wz, 2 * wy + 2 * xz,
                        2 * wz + 2 * xy, w2 - x2 + y2 - z2, 2 * yz - 2 * wx,
                        2 * xz - 2 * wy, 2 * wx + 2 * yz, w2 - x2 - y2 + z2],
                       dim=1).view(quat.size(0), 3, 3)


def annealing_weights(multires, ratio):
    alpha = ratio * multires
    out = []
    for ind in range(multires):
        w = (1. - np.cos(np.pi * min(max(alpha - float(ind), 0.), 1.))) / 2.
        out.extend([w, w])
    return out


def GMRobustError(x, c, square=False):
    if square:
        return 2. * x / (c * c) / (x / (c * c) + 4)
    return 2. * x * x / (c * c) / (x * x / (c * c) + 4)


def smpl_tmp_Apose(init_pose_type=0):
    pose = np.zeros((24, 3))
    leg, arm = {0: (10., 45.), 1: (7., 55.)}[init_pose_type]
    pose[1] = np.array([0, 0, leg / 180. * np.pi])
    pose[2] = np.array([0, 0, -leg / 180. * np.pi])
    pose[16] = np.array([0, 0, -arm / 180. * np.pi])
    pose[17] = np.array([0, 0, arm / 180. * np.pi])
    return pose.astype(np.float32)


def sample_points(pc_input, global_sigma, local_sigma, ratio=6):
    sample_size, dim = pc_input.shape
    sample_local = pc_input + (torch.randn_like(pc_input) * local_sigma)
    if ratio > 0:
        sample_global = (torch.rand(sample_size // ratio, dim, device=pc_input.device)
                         * (global_sigma * 2)) - global_sigma
        return torch.cat([sample_local, sample_global], dim=0)
    return sample_local


def compute_Jacobian(ps, ds, retain_graph, create_graph, allow_unused=False):
    """J[p, i, :] = d ds_i / d ps via three VJPs (autograd path, used when a graph is needed)."""
    rows = []
    ones = torch.ones_like(ds[..., 0])
    for i in range(3):
        keep = True if i < 2 else retain_graph
        out = torch.autograd.grad(ds[..., i], ps, ones, retain_graph=keep,
                                  create_graph=create_graph, allow_unused=allow_unused)
        rows.append(out[0].view(-1, 1, 3))
    return torch.cat(rows, dim=1)


def _fusable(deformer):
    return hasattr(deformer, "_fusable") and deformer._fusable()


def train_fused(deformer, sdf=None):
    """True when the training evaluations can run on the tensor-core training engine (train_ops.py)."""
    from selfreconcode_b200 import train_ops
    if not (train_ops.TC_TRAIN_ENABLED and _fusable(deformer) and hasattr(deformer, "forward_train")):
        return False
    return sdf is None or (hasattr(sdf, "_train_ok") and sdf._train_ok())


def mv3(M, v):
    """[P,3,3] x [P,3] without a GEMM launch."""
    return (M * v.unsqueeze(-2)).sum(-1)


def mtv3(M, v):
    """[P,3,3]^T x [P,3]."""
    return (M * v.unsqueeze(-1)).sum(-2)


def compute_deformed_normals(sdf, deformer, ps, defconds, batch_inds, ratio, phase):
    check = phase in ('train', 'Train')
    if not check and _fusable(deformer) and hasattr(sdf, "forward_fused"):
        # no graph requested: f, grad f, D, dD/dp from the fused forward-mode kernels
        _, onx, _ = sdf.forward_fused(ps, ratio, want_grad=True, want_feat=False)
        ds, grad_d_p, _ = deformer.forward_fused(ps, defconds, batch_inds, ratio, want_jac=True)
    elif check and train_fused(deformer, sdf):
        # training graph on the tensor-core engine: grad f and dD/dp are forward-mode OUTPUTS
        _, onx, _ = sdf.forward_train(ps, ratio, want_grad=True, want_feat=False)
        ds, grad_d_p = deformer.forward_train(ps, defconds, batch_inds, ratio, want_jac=True)
    else:
        sdfs = sdf(ps, ratio)
        onx = torch.autograd.grad(sdfs, ps, torch.ones_like(sdfs), retain_graph=check,
                                  create_graph=check)[0]
        ds = deformer(ps, defconds, batch_inds, ratio=ratio)
        grad_d_p = compute_Jacobian(ps, ds, check, check)
    grad_d_p_inv, inv_mask = FastDiff3x3MinvFunction.apply(grad_d_p)
    nx = mtv3(grad_d_p_inv, onx.view(-1, 3))
    n_inv_mask = ~inv_mask
    if n_inv_mask.sum().item() > 0:
        print('unwished error n_inv_mask:(%d:%d)' % (n_inv_mask.sum().item(), n_inv_mask.numel()))
        nnx = torch.zeros_like(nx)
        nnx[inv_mask] = nx[inv_mask]
        nnx[n_inv_mask] = mv3(grad_d_p[n_inv_mask], onx[n_inv_mask])
        nx = nnx
    nx = nx / nx.norm(dim=1, keepdim=True)
    return nx, ds


def deformed_normals_from(grad_f, J):
    """normalize(J^-T grad f) (fallback J grad f where J is singular) from already evaluated grad f [P,3] and
    dD/dp [P,3,3]: the no-graph core of compute_deformed_normals (utils/utils.py:139-152)."""
    with torch.no_grad():
        Jinv, ok = Fast3x3Minv(J.contiguous())
        nx = mtv3(Jinv, grad_f)
        nx = torch.where(ok.view(-1, 1), nx, mv3(J, grad_f))
        return nx / nx.norm(dim=1, keepdim=True)


def compute_cardinal_rays(deformer, ps, rays, defconds, batch_inds, ratio, phase):
    check = phase in ('train', 'Train')
    if not check and _fusable(deformer):
        ds, grad_d_p, _ = deformer.forward_fused(ps, defconds, batch_inds, ratio, want_jac=True)
    elif check and train_fused(deformer):
        ds, grad_d_p = deformer.forward_train(ps, defconds, batch_inds, ratio, want_jac=True)
    else:
        ds = deformer(ps, defconds, batch_inds, ratio=ratio)
        grad_d_p = compute_Jacobian(ps, ds, check, check)
    grad_d_p_inv, inv_mask = FastDiff3x3MinvFunction.apply(grad_d_p)
    crays = mv3(grad_d_p_inv, rays.view(-1, 3))
    n_inv_mask = ~inv_mask
    if n_inv_mask.sum().item() > 0:
        print('unwished error n_inv_mask:(%d:%d)' % (n_inv_mask.sum().item(), n_inv_mask.numel()))
        ncrays = torch.zeros_like(crays)
        ncrays[inv_mask] = crays[inv_mask]
        ncrays[n_inv_mask] = rays[n_inv_mask].detach()
        crays = ncrays
    crays = crays / crays.norm(dim=1, keepdim=True)
    return crays, ds


def compute_netRender_color(net, ps, ds, ns, vs, features, framefeatures, ratio):
    return net(ps, ns, vs, features, ratio)


def camera_normals(nx, R0):
    """The debug image's normal diag(-1,1,-1) R0^T n of every row of nx [P,3] (model/network.py:424)."""
    flip = torch.tensor([[-1., 0., 0.], [0., 1., 0.], [0., 0., -1.]], device=nx.device)
    return (flip @ R0.transpose(0, 1) @ nx.view(-1, 3, 1)).view(-1, 3)


def shade_rays(sdf, deformer, netRender, ps, rays, defconds, batch_inds, ratio, deformed_normals=False, cam_R0=None):
    """Everything the infer loop does with a traced point (model/network.py:356-368): template
    normal grad f / |grad f|, cardinal ray J^-1 v, rendered colour.  -> (normals, crays, rgb), no
    graph.  Large batches with the stock field modules run the SDF / translator sweeps (value +
    3 forward tangents), the pointwise geometry and the rendering network back to back on the
    tensor-core engine (ops.shade_and_render_tc); otherwise the per-op fused kernels are used.
    With `deformed_normals` a fourth output is the deformed-surface normal normalize(J^-T grad f) (the debug
    snapshot's, model/network.py:420-424), turned by camera_normals when a 3x3 `cam_R0` is given: on the
    tensor-core path it comes out of the same pointwise pass; otherwise from compute_deformed_normals(..., 'test')."""
    P = ps.shape[0]
    stock = (_fusable(deformer) and hasattr(sdf, "fused") and hasattr(netRender, "fused")
             and getattr(netRender, "mode", None) == 'idr' and getattr(netRender, "multires_n", 1) == 0
             and getattr(sdf, "d_out", 0) == 1)
    with torch.no_grad():
        if stock and ops.TC_ENABLED and P >= ops.TC_MIN_POINTS:
            tr, sk = deformer.defs[0], deformer.defs[1]
            full = sdf.fused()
            full.set_pe_weights(sdf._pe_weights(ratio['sdfRatio'] if isinstance(ratio, dict) else ratio))
            poses, trans = defconds[1]
            lbs = sk.lbs_state()
            lbs.set_pose(poses.view(poses.shape[0], 24, 3), trans)
            nfeat = full.desc.layer[full.desc.n_layers - 1].n - 1
            out = ops.shade_and_render_tc(full, tr.fused(ratio), lbs, netRender.fused(ratio), ps, rays, batch_inds,
                                          defconds[0], nfeat=nfeat, deformed_normals=deformed_normals, cam_R0=cam_R0)
            return (out[0], out[1], out[2], out[5]) if deformed_normals else out[:3]
        _, nx, feat = sdf.forward_fused(ps, ratio, want_grad=True, want_feat=True)
        nx = nx / nx.norm(dim=1, keepdim=True)
        crays, defVs = compute_cardinal_rays(deformer, ps, rays, defconds, batch_inds, ratio, 'test')
        rgb = compute_netRender_color(netRender, ps, defVs, nx, crays, feat, None, ratio)
        if not deformed_normals:
            return nx, crays, rgb
        dn, _ = compute_deformed_normals(sdf, deformer, ps, defconds, batch_inds, ratio, 'test')
        if cam_R0 is not None:
            dn = camera_normals(dn, cam_R0)
    return nx, crays, rgb, dn


# ------------------------------------------------------------------------------------------------
# Driver-facing helpers: what train.py / infer.py call on `utils` around the step
# (reference: utils/utils.py:174-316).  Plain torch; no third-party imports at module scope.
# ------------------------------------------------------------------------------------------------
def compute_face_areas(verts, faces):
    """verts [N,V,3], faces [F,3] or [N,F,3] -> triangle areas [N,F] (utils/utils.py:175-186)."""
    n = verts.shape[0]
    if faces.dim() == 2:
        faces = faces.unsqueeze(0).expand(n, -1, 3)
    assert faces.shape[0] == n and verts.shape[-1] == faces.shape[-1]
    tri = torch.gather(verts, 1, faces.reshape(n, -1, 1).expand(-1, -1, 3)).reshape(n, faces.shape[1], 3, 3)
    return torch.linalg.cross(tri[:, :, 1] - tri[:, :, 0], tri[:, :, 2] - tri[:, :, 0], dim=-1).norm(dim=-1) * 0.5


def compute_fnorms(verts, tri_fs):
    """Unit face normals; verts [V,3] or [B,V,3] (utils/utils.py:189-199)."""
    a, b, c = (verts.index_select(-2, tri_fs[:, i]) for i in range(3))
    n = torch.linalg.cross(b - a, c - a, dim=-1)
    return n / n.norm(2, -1, keepdim=True).clamp(min=1.e-6)


def compute_vnorms(verts, tri_fs, vertex_index, face_index):
    """Vertex normals as the normalised sum of incident face normals (utils/utils.py:224-230);
    `vertex_index[i]` / `face_index[i]` list every (vertex, incident face) pair."""
    fn = compute_fnorms(verts, tri_fs).index_select(-2, face_index)
    out = torch.zeros(verts.shape, dtype=verts.dtype, device=verts.device).index_add_(verts.dim() - 2, vertex_index, fn)
    return out / out.norm(2, -1, keepdim=True).clamp(min=1.e-6)


def DCTBasis(k, N):
    assert k < N
    n = torch.arange(N, dtype=torch.float64)
    scale = (1. / np.sqrt(float(N))) if k == 0 else np.sqrt(2. / float(N))
    return (torch.cos(np.pi * (n + 0.5) * k / float(N)) * scale).float()


def DCTNullSpace(k, N):
    """Rows k..N-1 of the orthonormal DCT-II basis: the temporal high-frequency space the pose
    trajectories are penalised in (model/network.py:585-593)."""
    return torch.stack([DCTBasis(i, N) for i in range(k, N)])


def DCTSpace(k, N):
    return torch.stack([DCTBasis(i, N) for i in range(0, k)])


def _new_engine(like, resolutions):
    from MCAcc import Seg3dLossless
    # the box as host lists (as getOptNet passes it): the engine builds its lattice tensors on the host first
    return Seg3dLossless(query_func=None, b_min=like.b_min.view(3).tolist(), b_max=like.b_max.view(3).tolist(),
                         resolutions=resolutions,
                         align_corners=False, balance_value=0.0, visualize=False, debug=False,
                         use_cuda_impl=False, faster=False).to(like.b_min.device)


def set_hierarchical_config(conf, name, optNet, dataloader, resolutions):
    """Switches the optimisation to hierarchy level `name` ('coarse' / 'medium' / 'fine'): new batch size,
    the level's loss / train config picked up at the next remesh, a new coarse-to-fine MC engine over the
    same box (utils/utils.py:237-256)."""
    from dataset.dataset import FrameLoader
    bs = conf.get_int('train.' + name + '.point_render.batch_size')
    dataloader = FrameLoader(dataloader.dataset, bs, sampler=dataloader.sampler, num_workers=dataloader.num_workers)
    optNet.next_conf = conf.get_config('loss_' + name)
    optNet.next_train_conf = conf.get_config('train.' + name)
    optNet.engine = _new_engine(optNet.engine, resolutions)
    return optNet, dataloader


def save_model(name, epoch, optNet, dataset):
    """`latest.pth` layout (utils/utils.py:257-264): epoch, model_state_dict, the camera tensors by
    their dataset names, per-frame poses / trans, shape, and the two latent-code tables."""
    out = {"epoch": epoch, "model_state_dict": optNet.state_dict()}
    out.update(dataset.camera_params)
    out.update({'poses': dataset.poses, 'trans': dataset.trans, 'shape': dataset.shape,
                'dcond': dataset.conds[0], 'rcond': dataset.conds[1]})
    torch.save(out, name)


def _cameras_from(dataset, n, device):
    from model.CameraMine import RectifiedPerspectiveCameras
    cam = dataset.camera_params
    return RectifiedPerspectiveCameras(cam['focal_length'].view(1, 2).expand(n, 2),
                                       cam['princeple_points'].view(1, 2).expand(n, 2),
                                       quat2mat(cam['cam2world_coord_quat'].view(1, 4)).expand(n, 3, 3),
                                       cam['world2cam_coord_trans'].view(1, 3).expand(n, 3),
                                       image_size=[(dataset.W, dataset.H)]).to(device)


def load_model(name, optNet, dataset, device, subsdfmodel=None, model_rm_prefix=None):
    """Inverse of save_model (utils/utils.py:266-316): engine buffers and the skin-weight volume are not
    restored (the volume comes from initial_skinner_*.pth), optional key-prefix removal, optional SDF
    substitution from a bare state_dict; dataset tensors keep their requires_grad flags."""
    saved = torch.load(name, map_location='cpu')
    state = {k: v for k, v in saved["model_state_dict"].items() if 'engine.' not in k}
    if model_rm_prefix:
        state = {k: v for k, v in state.items() if not any(k.startswith(p) for p in model_rm_prefix)}
    if subsdfmodel is not None:
        sub = torch.load(subsdfmodel, map_location='cpu')
        state = {k: v for k, v in state.items() if 'sdf.' not in k}
        state.update({'sdf.' + k: v for k, v in sub.items()})
    state = {k: v for k, v in state.items() if 'deformer.defs.1.ws' not in k}
    optNet.load_state_dict(state, strict=False)
    optNet = optNet.to(device)
    for i, key in enumerate(('dcond', 'rcond')):
        if key in saved:
            dataset.conds[i] = saved[key].requires_grad_()
    for key in ('poses', 'trans', 'shape'):
        keep = getattr(dataset, key).requires_grad
        setattr(dataset, key, saved[key].requires_grad_(keep))
        if key != 'shape':
            assert dataset.frame_num <= getattr(dataset, key).shape[0]
    dataset.camera_params = {k: saved[k].requires_grad_(v.requires_grad) for k, v in dataset.camera_params.items()}
    ras = optNet.maskRender.rasterizer
    n = getattr(ras.cameras, "_N", None) or ras.cameras.R.shape[0]
    ras.cameras = _cameras_from(dataset, n, device)
    return optNet, dataset
