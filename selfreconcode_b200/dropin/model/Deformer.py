"""Non-rigid deformation field: MLP offset + SMPL linear-blend skinning
(reference: model/Deformer.py:10-233) on the fused CUDA engines.

Class names, constructor signatures, buffers and state_dict keys follow the reference
(`defs.0.lin{l}.weight/bias`, `defs.1.{b_min,b_max,ws,Js,init_pose}`).  Without autograd the
whole composite D(p) = LBS(p + offset(p)) runs as ONE fused kernel (csrc/mlp_kernels.cu:
deform_kernel): PE + 5 layers + trilinear skin-weight lookup from a channels-last copy of the
volume + 24-bone blend, optionally with the analytic 3x3 Jacobian dD/dp.  With autograd the
same math runs as differentiable torch ops on the GPU, the sampler going through the drop-in
GridSamplerMine op (first and second order backward in csrc/grid_sampler.cu).
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from selfreconcode_b200 import ops
from .Embedder import get_embedder
from ._fused import FoldCache, needs_autograd, ratio_value, require_cuda, SR_ACT_NONE, SR_ACT_RELU


def _mm(a, b):
    """small trailing-dim matmul as broadcast multiply + sum (4x4 bone transforms): elementwise kernels only."""
    return (a.unsqueeze(-1) * b.unsqueeze(-3)).sum(-2)


def batch_rodrigues(theta):
    """axis-angle -> rotation (reference: smpl_pytorch/util.py:35-68), differentiable."""
    angle = torch.norm(theta + 1e-8, p=2, dim=1).unsqueeze(-1)
    normalized = theta / angle
    half = angle * 0.5
    quat = torch.cat([torch.cos(half), torch.sin(half) * normalized], dim=1)
    q = quat / quat.norm(p=2, dim=1, keepdim=True)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    w2, x2, y2, z2 = w * w, x * x, y * y, z * z
    wx, wy, wz, xy, xz, yz = w * x, w * y, w * z, x * y, x * z, y * z
    return torch.stack([w2 + x2 - y2 - z2, 2 * xy - 2 * wz, 2 * wy + 2 * xz,
                        2 * wz + 2 * xy, w2 - x2 + y2 - z2, 2 * yz - 2 * wx,
                        2 * xz - 2 * wy, 2 * wx + 2 * yz, w2 - x2 - y2 + z2],
                       dim=1).view(-1, 3, 3)


class CompositeDeformer(nn.Module):
    def __init__(self, deformers):
        super().__init__()
        self.N = len(deformers)
        self.defs = nn.ModuleList(deformers)

    def _fusable(self):
        return (self.N == 2 and isinstance(self.defs[0], MLPTranslator)
                and isinstance(self.defs[1], LBSkinner))

    def forward(self, ps, conds, batch_inds=None, **kwargs):
        assert self.N == len(conds)
        if self._fusable() and not isinstance(ps, list):
            tens = [ps, conds[0], conds[1][0], conds[1][1]] + list(self.defs[0].parameters())
            if not needs_autograd(*tens):
                d, _, _ = self.forward_fused(ps, conds, batch_inds, kwargs["ratio"], False)
                return d.view(ps.shape)
        out = ps
        for cond, deformer in zip(conds, self.defs):
            out = deformer(out, cond, batch_inds, **kwargs)
        return out

    def forward_train(self, ps, conds, batch_inds, ratio, want_jac=True):
        """Differentiable D(p) and (optionally) dD/dp on the tensor-core engine: the translator carries the
        point as value + 3 forward tangents (so d offset / dp is an output, utils/utils.py:106-120 without the
        three create_graph VJPs through the MLP); the LBS part and its 3x3 Jacobian go through the
        GridSamplerMine op and its double-backward kernels.  ps [P,3] with batch_inds, or [N,V,3] (mesh mode).
        -> (D(p) like ps, J [P,3,3] | None)"""
        from selfreconcode_b200 import train_ops as T
        import utils
        tr, sk = self.defs[0], self.defs[1]
        shape = ps.shape
        if batch_inds is None:
            n, v = ps.shape[0], ps.shape[1]
            cond_rows = conds[0].view(n, 1, -1).expand(n, v, conds[0].shape[-1]).reshape(n * v, -1)
        else:
            cond_rows = conds[0].index_select(0, batch_inds)
        pts = ps.reshape(-1, 3)
        off, Joff = tr.forward_train(pts, cond_rows, ratio, want_jac)
        tr.offset = off.view(shape)
        q = pts + off
        d = sk(q.view(shape), conds[1], batch_inds).reshape(-1, 3)
        if not want_jac:
            return d.view(shape), None
        Jl = utils.compute_Jacobian(q, d, True, True)                        # dLBS/dq via the sampler's backward ops
        eye = torch.eye(3, dtype=pts.dtype, device=pts.device).unsqueeze(0)
        return d.view(shape), T.small_matmul(Jl, eye + Joff)

    def forward_fused(self, ps, conds, batch_inds, ratio, want_jac=False, want_corner_idx=False):
        """-> (D(p) [P,3], J [P,3,3] | None, lbs corner indices | None); no graph.  Also sets
        defs[0].offset like the reference's MLPTranslator.forward does."""
        tr, sk = self.defs[0], self.defs[1]
        require_cuda(ps, "CompositeDeformer")
        net = tr.fused(ratio)
        poses, trans = conds[1]
        lbs = sk.lbs_state()
        lbs.set_pose(poses.view(poses.shape[0], 24, 3), trans)
        ppf = 0
        if batch_inds is None:
            ppf = ps.shape[1]
        d, off, jac, ci = ops.deform_forward(net, lbs, ps.reshape(-1, 3), batch_inds, conds[0],
                                             want_jac, True, want_corner_idx, ppf)
        tr.offset = off if batch_inds is not None else off.view(ps.shape[0], ps.shape[1], 3)
        return d, jac, ci


class MLPTranslator(nn.Module):
    def __init__(self, feature_vector_size, multires, weight_norm=False):
        super().__init__()
        dims = [3 + feature_vector_size, 512, 512, 512, 512, 3]
        self.feature_vector_size = feature_vector_size
        self.embed_fn = None
        self.multires = multires
        if multires > 0:
            self.embed_fn, input_ch = get_embedder(multires)
            dims[0] = input_ch + feature_vector_size
        self.num_layers = len(dims)
        for l in range(self.num_layers - 1):
            lin = nn.Linear(dims[l], dims[l + 1])
            if weight_norm:
                print('MLPTranslator:weight norm can influence weight initialization, can not '
                      'produce small weights as initialization. Now do not use weight_norm')
            if l == self.num_layers - 2:  # start from a (near) zero translation
                nn.init.normal_(lin.weight, mean=0.0, std=0.001)
                nn.init.constant_(lin.bias, 0.0)
            setattr(self, "lin" + str(l), lin)
        self.relu = nn.ReLU()
        self.offset = None
        self._cache = FoldCache()

    def fused(self, ratio):
        layers = []
        for l in range(self.num_layers - 1):
            lin = getattr(self, "lin" + str(l))
            layers.append(dict(v=lin.weight, g=None, b=lin.bias,
                               act=SR_ACT_RELU if l < self.num_layers - 2 else SR_ACT_NONE,
                               skip=False))
        params = [t for L in layers for t in (L["v"], L["b"])]
        dev = params[0].device
        require_cuda(params[0], "MLPTranslator")
        if self.multires <= 0:
            raise RuntimeError("MLPTranslator: the fused engine expects multires > 0")

        def build():
            return ops.FusedMLP(3 + 6 * self.multires + self.feature_vector_size, self.multires,
                                dev).fold(layers)

        net = self._cache.get(params, build)
        net.set_pe_weights(ops.annealing_weights(self.multires, ratio_value(ratio, "deformerRatio")))
        return net

    def forward_train(self, pts, cond_rows, ratio, want_jac=True):
        """pts [P,3], cond_rows [P,C] -> (offset [P,3], d offset / d p [P,3(m),3(c)] | None), differentiable
        w.r.t. pts, cond_rows and the parameters through the tensor-core training engine."""
        from selfreconcode_b200 import train_ops as T
        require_cuda(pts, "MLPTranslator.forward_train")
        ch = 4 if want_jac else 1
        L = self.num_layers - 1
        Ws = [getattr(self, "lin" + str(l)).weight for l in range(L)]
        bs = [getattr(self, "lin" + str(l)).bias for l in range(L)]
        acts = [SR_ACT_RELU] * (L - 1) + [SR_ACT_NONE]
        d_in = 3 + 6 * self.multires + self.feature_vector_size
        pe_w = ops.annealing_weights(self.multires, ratio_value(ratio, "deformerRatio"))
        x0 = T.embed_rows(pts, self.multires, pe_w, ch, extra=cond_rows)
        packs = ops.tc_net(self.fused(ratio)).layers
        out = T.tc_mlp(x0, T.MlpConfig(acts, [False] * L, d_in, ch, packs), Ws, bs).view(pts.shape[0], ch, 3)
        off = out[:, 0]
        jac = out[:, 1:].transpose(1, 2) if want_jac else None      # [P, m, c] = d off_m / d p_c
        return off, jac

    def forward(self, ps, conds, batch_inds=None, **kwargs):
        require_cuda(ps, "MLPTranslator.forward")
        if not needs_autograd(ps, conds, *self.parameters()):
            net = self.fused(kwargs["ratio"])
            ppf = 0 if batch_inds is not None else ps.shape[1]
            d, off, _, _ = ops.deform_forward(net, None, ps.reshape(-1, 3), batch_inds, conds,
                                              False, True, False, ppf)
            if batch_inds is not None:
                self.offset = off
                return d
            self.offset = off.view(ps.shape[0], ps.shape[1], 3)
            return d.view(ps.shape[0], ps.shape[1], 3)
        ratio = ratio_value(kwargs['ratio'], 'deformerRatio')
        if self.embed_fn is not None:
            if ratio is None:
                ps = self.embed_fn(ps)
            elif ratio <= 0:
                ps = self.embed_fn(ps, [0.0] * (self.multires * 2))
            else:
                ws = [w for w in ops.annealing_weights(self.multires, ratio) for _ in (0, 1)]
                ps = self.embed_fn(ps, ws)
        if batch_inds is not None:
            x = torch.cat([ps, conds.index_select(0, batch_inds)], dim=1)
        else:
            c = conds.view(-1, 1, self.feature_vector_size).expand(-1, ps.shape[1], -1)
            x = torch.cat([ps, c], dim=-1).view(-1, ps.shape[-1] + self.feature_vector_size)
        for l in range(self.num_layers - 1):
            x = getattr(self, "lin" + str(l))(x)
            if l < self.num_layers - 2:
                x = self.relu(x)
        if batch_inds is not None:
            self.offset = x
            return ps[..., :3] + x
        self.offset = x.view(ps.shape[0], ps.shape[1], 3)
        return ps[..., :3] + self.offset


def getTranslatorNet(device, conf):
    if 'type' in conf:
        return globals()[conf.get_string('type')](conf.get_int('condlen'),
                                                  multires=conf.get_int('multires')).to(device)
    return MLPTranslator(conf.get_int('condlen'), multires=conf.get_int('multires')).to(device)


class LBSkinner(nn.Module):
    """SMPL-skeleton LBS with a trilinear skin-weight volume (Deformer.py:86-233)."""

    def __init__(self, ws, bmins, bmaxs, Js, parents, init_pose=None, align_corners=False):
        super().__init__()

        def as_buf(v):
            if isinstance(v, list):
                return torch.tensor(v, dtype=torch.float).view(1, 3)
            if isinstance(v, np.ndarray):
                return torch.from_numpy(v.astype(np.float32)).view(1, 3)
            return v.view(1, 3)

        self.register_buffer('b_min', as_buf(bmins))
        self.register_buffer('b_max', as_buf(bmaxs))
        if isinstance(ws, np.ndarray):
            ws = torch.from_numpy(ws.astype(np.float32))
        self.register_buffer('ws', ws.to(torch.float))
        self.align_corners = align_corners
        assert align_corners == False
        self.register_buffer('Js', Js.view(24, 3))
        self.parents = parents
        if init_pose is None:
            self.register_buffer('init_pose', None)
        else:
            if isinstance(init_pose, np.ndarray):
                init_pose = torch.from_numpy(init_pose.astype(np.float32))
            if init_pose.numel() == 24 * 3:
                self.init_pose_inverse(batch_rodrigues(init_pose.view(-1, 3)).view(24, 3, 3), self.Js)
            else:
                self.register_buffer('init_pose', init_pose.view(24, 4, 4))
        self._lbs = None
        self._lbs_sig = None

    def init_pose_inverse(self, init_pose, Js):
        Rs, Ts = [init_pose[0]], [Js[0]]
        for i in range(1, self.parents.shape[0]):
            p = int(self.parents[i])
            Rs.append(Rs[p].matmul(init_pose[i]))
            Ts.append(Rs[p].matmul((Js[i] - Js[p]).view(-1, 1)).view(-1) + Ts[p])
        invs = []
        for R, T in zip(Rs, Ts):
            inv = torch.zeros(4, 4, dtype=R.dtype, device=R.device)
            inv[3, 3] = 1.0
            inv[:3, :3] = R.transpose(0, 1)
            inv[:3, 3] = (-T.view(1, -1).matmul(R)).view(-1)
            invs.append(inv)
        self.register_buffer('init_pose', torch.stack(invs, dim=0))

    def lbs_state(self):
        """Device-side state for the fused path (channels-last volume, rebuilt if `ws` changes)."""
        require_cuda(self.ws, "LBSkinner")
        sig = (self.ws.data_ptr(), self.ws._version, self.b_min.data_ptr(), self.b_min._version,
               self.b_max.data_ptr(), self.b_max._version, self.Js.data_ptr(), self.Js._version,
               None if self.init_pose is None else (self.init_pose.data_ptr(), self.init_pose._version))
        if self._lbs is None or sig != self._lbs_sig:
            self._lbs = ops.LbsState(self.ws, self.b_min, self.b_max, self.Js,
                                     [int(p) for p in self.parents], self.init_pose)
            self._lbs_sig = sig
        return self._lbs

    def _chain(self, poses):
        batch_size = poses.shape[0]
        R = batch_rodrigues(poses.view(-1, 3)).view(batch_size, 24, 3, 3)
        Js = self.Js.view(1, 24, 3, 1).expand(batch_size, 24, 3, 1)

        def make_A(Rm, t):
            R_homo = F.pad(Rm, [0, 0, 0, 1, 0, 0])
            t_homo = torch.cat([t, torch.ones(batch_size, 1, 1, device=Rm.device)], dim=1)
            return torch.cat([R_homo, t_homo], 2)

        results = [make_A(R[:, 0], Js[:, 0])]
        for i in range(1, self.parents.shape[0]):
            p = int(self.parents[i])
            results.append(_mm(results[p], make_A(R[:, i], Js[:, i] - Js[:, p])))
        return torch.stack(results, dim=1), Js

    def posedSkeleton(self, conds):
        poses, trans = conds
        assert poses.shape[0] == trans.shape[0]
        if not needs_autograd(poses):
            require_cuda(poses, "LBSkinner.posedSkeleton")
            lbs = self.lbs_state()
            return lbs.set_pose(poses.reshape(poses.shape[0], 24, 3), trans, want_posed_joints=True)
        results, _ = self._chain(poses)
        return results[:, :, :3, 3]

    def forward(self, ps, conds, batch_inds=None, **kwargs):
        from MCAcc import GridSamplerMine3dFunction
        if isinstance(ps, list):
            tps, ps = ps
        else:
            tps = ps
        poses, trans = conds
        batch_size = poses.shape[0]
        assert batch_size == trans.shape[0]
        require_cuda(ps, "LBSkinner.forward")
        results, Js = self._chain(poses)
        if self.init_pose is None:
            Js_w0 = torch.cat([Js, torch.zeros(batch_size, 24, 1, 1, device=poses.device)], dim=2)
            init_bone = F.pad(_mm(results, Js_w0), [3, 0, 0, 0, 0, 0, 0, 0])
            A = results - init_bone
        else:
            A = _mm(results, self.init_pose.view(1, 24, 4, 4).expand(batch_size, 24, 4, 4))
        nps = 2. * (tps.reshape(-1, 3) - self.b_min) / (self.b_max - self.b_min) - 1.
        ps_ws = GridSamplerMine3dFunction.apply(self.ws, nps.reshape(1, 1, 1, -1, 3)) \
            .view(-1, nps.shape[0]).transpose(0, 1)
        if batch_inds is None:
            _, pnum, _ = ps.shape
            ps_ws = ps_ws.view(batch_size, pnum, 24)
            T = (ps_ws.unsqueeze(-1) * A.view(batch_size, 1, 24, 16)).sum(2).view(batch_size, pnum, 4, 4)
            ph = torch.cat([ps, torch.ones(batch_size, pnum, 1, device=ps.device)], dim=2)
            return (T[:, :, :3, :] * ph.unsqueeze(-2)).sum(-1) + trans.view(-1, 1, 3)
        ps = ps.reshape(-1, 3)
        assert batch_inds.numel() == ps.shape[0]
        # one gather instead of the reference's per-frame masked loop with a host sync per frame
        # (Deformer.py:226-231): T_p = sum_j w_pj A[b_p, j]
        # (broadcast multiply + sum instead of einsum / matmul: no cuBLAS launches in the training step)
        T = (ps_ws.unsqueeze(-1) * A.view(batch_size, 24, 16).index_select(0, batch_inds)).sum(1).view(-1, 4, 4)
        v = (T[:, :3, :] * F.pad(ps, (0, 1), mode='constant', value=1).unsqueeze(-2)).sum(-1)
        return v + trans.index_select(0, batch_inds)


def smooth_weights(weights, times=3):
    """The Deformer-module variant of the volume smoother (model/Deformer.py:234-244): same damped
    6-neighbour pass as utils.LBSWsmpl.smooth_weights but WITHOUT zeroing small weights."""
    for _ in range(times):
        c = weights[:, :, 1:-1, 1:-1, 1:-1]
        mean = (weights[:, :, 2:, 1:-1, 1:-1] + weights[:, :, :-2, 1:-1, 1:-1] +
                weights[:, :, 1:-1, 2:, 1:-1] + weights[:, :, 1:-1, :-2, 1:-1] +
                weights[:, :, 1:-1, 1:-1, 2:] + weights[:, :, 1:-1, 1:-1, :-2]) / 6.0
        weights[:, :, 1:-1, 1:-1, 1:-1] = (c - mean) * 0.7 + mean
        weights = weights / weights.sum(1, keepdim=True)
    return weights


smooth_weights.lbsw_cut = 0.0


def compute_lbswField(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners=False,
                      mean_neighbor=5, smooth_times=30):
    """model/Deformer.py:246-284 (the copy getOptNet's initialiser uses: no small-weight cut)."""
    from utils.LBSWsmpl import compute_lbswField as _field
    return _field(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners, mean_neighbor,
                  smooth_times, smooth=smooth_weights)


def initialLBSkinner(gender, shape, pose, resolution, bmins=None, bmaxs=None):
    """One-time construction of the LBS field from the SMPL body model (model/Deformer.py:286-296):
    posed template vertices -> (adaptive) box -> 30-NN skin-weight volume -> LBSkinner.
    Needs the reference's `smpl_pytorch` package and the SMPL model files (licensed assets,
    not part of this repository): imported lazily so the module loads without them."""
    from smpl_pytorch.SMPL import getSMPL
    smpl = getSMPL(gender).to(shape.device)
    Js, _ = smpl.skeleton(shape.view(1, -1), True)
    verts, _, _ = smpl(shape.view(1, -1), pose.view(1, 24, 3), True)
    if bmins is None or bmaxs is None:
        margin = np.array([0.15, 0.15, 0.20], dtype=np.float32)
        bmins = (verts[0].min(0)[0].cpu().numpy() - margin).tolist()
        bmaxs = (verts[0].max(0)[0].cpu().numpy() + margin).tolist()
    ws = compute_lbswField(bmins, bmaxs, resolution, verts.view(6890, 3), smpl.weight.view(6890, 24),
                           align_corners=False, mean_neighbor=30, smooth_times=30)
    skinner = LBSkinner(ws, bmins, bmaxs, Js, smpl.parents, init_pose=pose, align_corners=False)
    return skinner, verts.view(6890, 3), torch.tensor(smpl.faces, dtype=torch.long, device=verts.device)
