"""Per-step orchestration of the hot path (reference: model/network.py:149-814, OptimNetwork).

What is mirrored, with the reference's names and call conventions:
  * `discretizeSDF`            network.py:292-302  coarse-to-fine SDF grid + marching cubes
  * `infer` (ray part) as `infer_rays`   :342-372  trace + shade every foreground ray of N frames
  * `forward` (ray part) as `forward_rays` :509-644  trace, eikonal, colour and normal losses
  * `propagateTmpPsGrad`       :702-814  implicit differentiation of {f(p)=0, (D(p)-c) x v = 0}
`forward()` / `infer()` themselves start with a pytorch3d mesh / point rasterisation of the deformed
template (network.py:485-505, 317-345) that seeds `FindSurfacePs`; that seed is out of scope
(SURVEY.md section 8f-1), so here they take the seed (batch/row/col indices + start points) from the
caller or from an injected `raster_seed` callable and then run exactly the reference's sequence.
No-grad evaluations run on the fused kernels; losses that need a graph use the modules' autograd
path (same math as torch ops on the GPU).
"""
import os
import os.path as osp

import numpy as np
import torch
import torch.nn as nn

import utils
from FastMinv import Fast3x3Minv
import MCGpu
from selfreconcode_b200 import ops
from .CameraMine import RectifiedPerspectiveCameras, PointsRendererWithFrags
from ._fused import scatter_rows


def _p3d():
    """pytorch3d pieces the mesh / point-cloud silhouette part of the step uses (network.py:121-143).
    Imported on first use: the per-point hot path never needs them."""
    import types
    try:
        from pytorch3d.structures import Meshes, Pointclouds
        from pytorch3d.loss import mesh_edge_loss, mesh_laplacian_smoothing, mesh_normal_consistency
        from pytorch3d.renderer import (RasterizationSettings, MeshRasterizer, SoftSilhouetteShader, TexturesVertex,
                                        PointsRasterizationSettings, PointsRasterizer, PointLights, AlphaCompositor)
        from pytorch3d.renderer.mesh.renderer import MeshRendererWithFragments
    except ImportError as e:  # pragma: no cover - depends on the installation
        raise RuntimeError("this part of OptimNetwork needs pytorch3d (mesh / point rasterisers, mesh losses): " +
                           str(e))
    return types.SimpleNamespace(**{k: v for k, v in locals().items() if k not in ("types", "e")})


def vertex_face_pairs(faces, n_verts):
    """(vertex id, incident face id) pairs, vertex-major: what the reference extracts from openmesh's
    vertex_face_indices() (network.py:472-477) -- here one device sort of the face table."""
    flat = faces.reshape(-1)
    order = torch.argsort(flat, stable=True)
    return flat[order], torch.div(order, 3, rounding_mode='floor')


def _scatter_mean(src, index, n):
    """torch_scatter.scatter(..., reduce='mean', dim_size=n) (network.py:617,637), summed in a fixed order so that the
    step's loss is bit-identical from run to run."""
    s = scatter_rows(src, index, n)
    c = scatter_rows(torch.ones_like(index, dtype=src.dtype), index, n).clamp(min=1)
    return s / c.view((-1,) + (1,) * (src.dim() - 1))


def _cross_matrix(v):
    m = torch.zeros(v.shape[0], 3, 3, dtype=v.dtype, device=v.device)
    m[:, 0, 1], m[:, 0, 2] = -v[:, 2], v[:, 1]
    m[:, 1, 0], m[:, 1, 2] = v[:, 2], -v[:, 0]
    m[:, 2, 0], m[:, 2, 1] = -v[:, 1], v[:, 0]
    return m


class OptimNetwork(nn.Module):
    def __init__(self, TmpSdf, Deformer, accEngine, maskRender, netRender, conf=None):
        super().__init__()
        self.conf = conf
        self.sdf = TmpSdf
        self.deformer = Deformer
        self.maskRender = maskRender
        self.netRender = netRender
        self.engine = accEngine
        cams = maskRender.rasterizer.cameras if maskRender is not None else None
        self.angThred = cams.angThreshold(0.5) if cams is not None else 0.02
        self.TmpVs = None
        self.Tmpfs = None
        self.forward_time = 0
        self.remesh_intersect = 30
        self.remesh_time = 0.
        self.next_conf = None
        self.next_train_conf = None
        self.pcRender = None
        self.draw = False
        self.enable_mesh_color = True
        self.sdfShrinkRadius = 0.0
        self.info = {}
        self.TmpPs = None
        self.mesh_reg_topo = None  # ops.MeshRegTopology of Tmpfs, built when a mesh regulariser weight is positive
        self.raster_seed = None   # callable(frame_ids, TmpVs, Tmpfs, defconds, ratio) -> seed dict

    # ---- differentiable value-only evaluations (tensor-core training engine when the modules are the stock ones)
    def _sdf_value(self, pts, ratio):
        if utils.train_fused(self.deformer, self.sdf):
            return self.sdf.forward_train(pts, ratio, want_grad=False, want_feat=False)[0]
        return self.sdf(pts, ratio)

    def _deform(self, ps, conds, batch_inds, ratio):
        if utils.train_fused(self.deformer):
            return self.deformer.forward_train(ps, conds, batch_inds, ratio, want_jac=False)[0]
        return self.deformer(ps, conds, batch_inds, ratio=ratio)

    def _offset(self, ps, d_cond, ratio):
        """translator offsets in mesh mode ps [N,M,3] (network.py:553, 571)."""
        tr = self.deformer.defs[0]
        if utils.train_fused(self.deformer):
            n, m = ps.shape[0], ps.shape[1]
            cr = d_cond.view(n, 1, -1).expand(n, m, d_cond.shape[-1]).reshape(n * m, -1)
            off, _ = tr.forward_train(ps.reshape(-1, 3), cr, ratio, want_jac=False)
            tr.offset = off.view(n, m, 3)
            return tr.offset
        tr(ps, d_cond, ratio=ratio)
        return tr.offset

    # ---- cameras ----------------------------------------------------------------------------
    def _cameras(self, n, device):
        focals, pps, Rs, Ts, H, W = self.dataset.get_camera_parameters(n, device)
        return RectifiedPerspectiveCameras(focals, pps, Rs, Ts, image_size=[(W, H)]).to(device), H, W

    # ---- network.py:172-205 -------------------------------------------------------------------
    def update_hierarchical_config(self, device):
        """Applies the hierarchy level queued by utils.set_hierarchical_config at the next remesh: new loss
        conf, point renderer with the level's radius, hard (blur 0) silhouette rasteriser settings.  With the
        built-in mesh rasteriser (raster.MeshRasterizer) the point renderer is the built-in device one and no
        pytorch3d is needed; with pytorch3d's rasteriser it is pytorch3d's."""
        if self.next_conf is None:
            return
        self.conf = self.next_conf
        self.forward_time = 0
        tc = self.next_train_conf
        self.remesh_intersect = tc.get_int('point_render.remesh_intersect')
        self.sdfShrinkRadius = 0.0
        ras = self.maskRender.rasterizer if self.maskRender is not None else None
        from . import raster
        if isinstance(ras, raster.MeshRasterizer):
            H, W = ras.raster_settings.image_size[0], ras.raster_settings.image_size[1]
            self.pcRender = raster.PointsSilhouetteRenderer(raster.PointsRasterizer(
                cameras=ras.cameras, raster_settings=raster.PointsRasterizationSettings(
                    image_size=(H, W), radius=tc.get_float('point_render.radius'), points_per_pixel=50))).to(device)
            ras.raster_settings = raster.RasterSettings((H, W))
        elif ras is not None and hasattr(ras, "raster_settings"):
            P = _p3d()
            H, W = ras.raster_settings.image_size[0], ras.raster_settings.image_size[1]
            big = 92 if 1024 < max(H, W) <= 2048 else None
            self.pcRender = PointsRendererWithFrags(
                rasterizer=P.PointsRasterizer(cameras=ras.cameras, raster_settings=P.PointsRasterizationSettings(
                    image_size=(H, W), radius=tc.get_float('point_render.radius'), bin_size=big,
                    points_per_pixel=50)),
                compositor=P.AlphaCompositor(background_color=None)).to(device)
            ras.raster_settings = P.RasterizationSettings(
                image_size=(H, W), blur_radius=0., bin_size=big, faces_per_pixel=1, perspective_correct=True,
                clip_barycentric_coords=False, cull_backfaces=ras.raster_settings.cull_backfaces)
        self.next_conf = None
        self.next_train_conf = None

    # ---- network.py:207-290 -------------------------------------------------------------------
    def initializeTmpSDF(self, nepochs, save_name, with_normals=False):
        """IGR pre-fit of the SDF to the SMPL template (points `tmpBodyVs`, optional normals): |f| on the
        surface + 0.1 eikonal on jittered / uniform samples (+ normal term), Adam lr 5e-3 halved every 500
        epochs, 5000-point batches; all PE bands off (ratio -1)."""
        net = self.sdf
        net.train()
        opt = torch.optim.Adam([{"params": net.parameters(), "lr": 0.005, "weight_decay": 0}])
        sched = torch.optim.lr_scheduler.StepLR(opt, 500, 0.5)
        vs = self.tmpBodyVs
        ns = getattr(self, "tmpBodyNs", None)
        with_normals = bool(with_normals and ns is not None)
        if not with_normals:
            ns = torch.ones_like(vs) / np.sqrt(3)
        for epoch in range(1, nepochs + 1):
            perm = torch.randperm(vs.shape[0])
            batches = list(zip(torch.split(vs[perm], 5000), torch.split(ns[perm], 5000)))
            for bi, (on_pts, normals) in enumerate(batches):
                off_pts = utils.sample_points(on_pts, 1.8, 0.01)
                loss, mnfld_loss, grad_loss, normals_loss = self.igr_losses(on_pts, off_pts, normals, with_normals)
                opt.zero_grad()
                loss.backward()
                opt.step()
                if bi == len(batches) - 1:
                    print('Train Epoch: {}\tTrain Loss: {:.6f}\tManifold loss: {:.6f}\tGrad loss: {:.6f}'
                          '\tNormals Loss: {:.6f}'.format(epoch, loss.item(), mnfld_loss.item(), grad_loss.item(),
                                                          normals_loss.item()))
            sched.step()
        if save_name:
            torch.save(net.state_dict(), save_name)

    def igr_losses(self, on_pts, off_pts, normals, with_normals):
        """One IGR batch -> (loss, manifold, eikonal, normal term) (network.py:243-270).  With the stock SDF module the
        on- and off-surface points go through ONE tensor-core forward_train call with grad f as a forward-mode output,
        so loss.backward() is one reverse sweep plus the weight-gradient GEMMs; otherwise the reference's autograd
        loop (create_graph=True, then a double backward)."""
        net = self.sdf
        n_on = on_pts.shape[0]
        if hasattr(net, "_train_ok") and net._train_ok():
            f, g, _ = net.forward_train(torch.cat([on_pts.detach(), off_pts.detach()]), -1, want_grad=True,
                                        want_feat=False)
            on_pred, on_grad, off_grad = f[:n_on], g[:n_on], g[n_on:]
        else:
            on_pts = on_pts.detach().requires_grad_()
            off_pts = off_pts.detach().requires_grad_()
            on_pred = net(on_pts, -1)
            off_pred = net(off_pts, -1)
            on_grad = net.gradient(on_pts, on_pred)
            off_grad = net.gradient(off_pts, off_pred)
        mnfld_loss = on_pred.abs().mean()
        grad_loss = ((off_grad.norm(2, dim=-1) - 1) ** 2).mean()
        loss = mnfld_loss + 0.1 * grad_loss
        if with_normals:
            normals_loss = (on_grad - normals.view(-1, 3).to(on_grad.dtype)).abs().norm(2, dim=1).mean()
            loss = loss + 1.0 * normals_loss
        else:
            normals_loss = torch.zeros(1)
        return loss, mnfld_loss, grad_loss, normals_loss

    # ---- network.py:292-302 -------------------------------------------------------------------
    def discretizeSDF(self, ratio, engine=None, balance_value=0.):
        sdf = self.sdf

        def query_func(points):
            with torch.no_grad():
                if hasattr(sdf, "forward_fused"):  # value only: skip the 256-d feature head
                    return sdf.forward_fused(points.reshape(-1, 3), ratio, False, False,
                                             refine_about=balance_value)[0].reshape(1, 1, -1)
                return sdf.forward(points.reshape(-1, 3), ratio).reshape(1, 1, -1)

        if engine is None:
            engine = self.engine
        engine.balance_value = balance_value
        engine.query_func = query_func
        sdfs = engine.forward()
        verts, faces = MCGpu.mc_gpu(sdfs[0, 0].permute(2, 1, 0).contiguous(), engine.spacing_x,
                                    engine.spacing_y, engine.spacing_z, engine.bx, engine.by, engine.bz,
                                    balance_value)
        return verts, faces

    # ---- ray part of infer(): network.py:342-372 ------------------------------------------------
    def infer_rays(self, batch_inds, row_inds, col_inds, initTmpPs, H, W, ratio, frame_ids, chunk=1 << 18):
        device = initTmpPs.device
        N = frame_ids.numel()
        cameras, _, _ = self._cameras(N, device)
        poses, trans, d_cond, rendcond = self.dataset.get_grad_parameters(frame_ids, device)
        pix = torch.cat([col_inds.view(-1, 1), row_inds.view(-1, 1), torch.ones_like(col_inds.view(-1, 1))], dim=-1)
        with torch.no_grad():
            rays = cameras.view_rays(pix.float())
        defconds = [d_cond.detach(), [poses.detach(), trans.detach()]]
        tcolors = []
        cam_pos = cameras.cam_pos().detach()
        for rays_, ps_, bi_ in zip(torch.split(rays, chunk), torch.split(initTmpPs, chunk), torch.split(batch_inds, chunk)):
            ps_, check = utils.OptimizeSurfacePs(cam_pos, rays_.detach(), ps_.clone(), bi_, self.sdf, ratio,
                                                 self.deformer, defconds, dthreshold=1.e-4, athreshold=self.angThred,
                                                 w1=3.05, w2=1., times=30)
            if hasattr(self.sdf, "forward_fused"):
                tcolors.append(utils.shade_rays(self.sdf, self.deformer, self.netRender, ps_, rays_, defconds, bi_,
                                                ratio)[2])
                continue
            ps_ = ps_.detach().requires_grad_(True)   # user-supplied field modules: reference sequence
            sdfs = self.sdf(ps_, ratio)
            nx = torch.autograd.grad(sdfs, ps_, torch.ones_like(sdfs))[0]
            nx = nx / nx.norm(dim=1, keepdim=True)
            crays, defVs = utils.compute_cardinal_rays(self.deformer, ps_, rays_, defconds, bi_, ratio, 'test')
            with torch.no_grad():
                self.sdf(ps_, ratio)
                tcolors.append(utils.compute_netRender_color(self.netRender, ps_, defVs, nx, crays,
                                                             self.sdf.rendcond, None, ratio))
        tcolors = torch.clamp((torch.cat(tcolors, dim=0) / 2. + 0.5) * 255., min=0., max=255.)
        colors = torch.ones(N, H, W, 3, device=device) * 255.
        colors[batch_inds, row_inds, col_inds, :] = tcolors
        return colors

    # ---- ray part of forward(): network.py:509-644 ----------------------------------------------
    def forward_rays(self, datas, batch_inds, row_inds, col_inds, initTmpPs, ratio, frame_ids,
                     extra_points=None, count_step=True):
        """Loss terms that depend on rays: eikonal (grad_weight), colour, normal.  `extra_points`
        stands for the template vertices the reference adds to the eikonal sample set (:543)."""
        device = frame_ids.device
        conf = self.conf
        if getattr(self.sdf, "_weff", None) is not None:
            self.sdf._weff = None        # a previous call that raised must not leave its weight sub-graph behind
        gtCs = datas['img'].to(device)
        N = gtCs.shape[0]
        cameras, H, W = self._cameras(N, device)
        pix = torch.cat([col_inds.view(-1, 1), row_inds.view(-1, 1), torch.ones_like(col_inds.view(-1, 1))], dim=-1)
        rays = cameras.view_rays(pix.float())
        poses, trans, d_cond, rendcond = self.dataset.get_grad_parameters(frame_ids, device)
        defconds = [d_cond, [poses, trans]]
        self.info = {}
        initTmpPs, check = utils.OptimizeSurfacePs(cameras.cam_pos().detach(), rays.detach(), initTmpPs, batch_inds,
                                                   self.sdf, ratio, self.deformer, defconds, dthreshold=5.e-5,
                                                   athreshold=self.angThred, w1=3.05, w2=1., times=10)
        self.info['rayInfo'] = (check.numel(), check.sum().item())
        self.TmpPs = None
        total_loss = torch.zeros((), device=device)
        # eikonal on jittered surface points + uniform samples (:543-549)
        base = initTmpPs if extra_points is None else torch.cat([initTmpPs, extra_points.detach()], dim=0)
        nonmnfld_pnts = utils.sample_points(base, 1.8, 0.01)
        nonmnfld_pnts.requires_grad_()
        fused_train = utils.train_fused(self.deformer, self.sdf) and self.netRender._train_ok() \
            if hasattr(self.netRender, "_train_ok") else False
        import contextlib
        shared = self.sdf.shared_weights() if fused_train else contextlib.nullcontext()
        shared.__enter__()       # eikonal and surface-point evaluations share one weight-norm sub-graph
        if fused_train:
            # eikonal term on the tensor-core training engine: grad f is a forward-mode output (network.py:545-547)
            _, grad, _ = self.sdf.forward_train(nonmnfld_pnts, ratio, want_grad=True, want_feat=False)
        else:
            pred = self.sdf(nonmnfld_pnts, ratio)
            grad = self.sdf.gradient(nonmnfld_pnts, pred)
        grad_loss = ((grad.norm(2, dim=-1) - 1) ** 2).mean()
        self.info['grad_loss'] = grad_loss.item()
        total_loss = total_loss + grad_loss * conf.get_float('grad_weight')
        total_loss = total_loss + self._regularisers(nonmnfld_pnts, base, N, d_cond, poses, trans, ratio, frame_ids)
        self.info['color_loss'] = -1.0
        self._tmp_geom = None
        if self.info['rayInfo'][1] > 0:
            self.TmpPs = initTmpPs[check]
            self.TmpPs.requires_grad = True
            self.rays = rays[check]
            self.batch_inds = batch_inds[check]
            self.col_inds = col_inds[check]
            self.row_inds = row_inds[check]
            grad_d_p = None
            if fused_train:
                # f, grad f, rendcond in one forward-mode sweep; D(p), dD/dp in another (network.py:606-610)
                sdfs, gf_raw, rendcond_p = self.sdf.forward_train(self.TmpPs, ratio, want_grad=True, want_feat=True)
                self.sdf.rendcond = rendcond_p
                nx = gf_raw / gf_raw.norm(dim=1, keepdim=True)
                defVs, grad_d_p = self.deformer.forward_train(self.TmpPs, defconds, self.batch_inds, ratio, True)
                # grad f and dD/dp at the surface points, reused (detached) by the normal weights below and by
                # propagateTmpPsGrad: the reference re-evaluates both there (network.py:625, 721-748)
                self._tmp_geom = (self.TmpPs, gf_raw.detach(), grad_d_p.detach())
                Jinv, inv_mask = utils.FastDiff3x3MinvFunction.apply(grad_d_p)
                crays = utils.mv3(Jinv, self.rays.view(-1, 3))
                crays = torch.where(inv_mask.view(-1, 1), crays, self.rays.detach())
                crays = crays / crays.norm(dim=1, keepdim=True)
            else:
                sdfs = self.sdf(self.TmpPs, ratio)
                nx = torch.autograd.grad(sdfs, self.TmpPs, torch.ones_like(sdfs), retain_graph=True,
                                         create_graph=True)[0]
                nx = nx / nx.norm(dim=1, keepdim=True)
                crays, defVs = utils.compute_cardinal_rays(self.deformer, self.TmpPs, self.rays, defconds,
                                                           self.batch_inds, ratio, 'train')
            if conf.get_float('color_weight') > 0.:
                colors = utils.compute_netRender_color(self.netRender, self.TmpPs, defVs, nx, crays, self.sdf.rendcond,
                                                       None, ratio)
                color_loss = (gtCs[self.batch_inds, self.row_inds, self.col_inds, :] - colors).abs().sum(1)
                color_loss = _scatter_mean(color_loss, self.batch_inds, N).mean()
                self.info['color_loss'] = color_loss.item()
                total_loss = total_loss + conf.get_float('color_weight') * color_loss
            if 'normal' in datas and 'normal_weight' in conf and conf.get_float('normal_weight') > 0.:
                if 'weighted_normal' in conf and conf.get_bool('weighted_normal'):
                    if self._tmp_geom is not None:
                        cnx = utils.deformed_normals_from(self._tmp_geom[1], self._tmp_geom[2])
                    else:
                        cnx, _ = utils.compute_deformed_normals(self.sdf, self.deformer, self.TmpPs, defconds,
                                                                self.batch_inds, ratio, 'test')
                    weights = torch.clamp((-self.rays * cnx.detach()).sum(1).detach(), max=1., min=0.) ** 2
                else:
                    weights = torch.ones(nx.shape[0], device=device)
                gtn = datas['normal'].to(device)[self.batch_inds, self.row_inds, self.col_inds, :]
                flip = torch.tensor([[-1., 0., 0.], [0., 1., 0.], [0., 0., -1.]], device=device)
                gtn = utils.mv3((cameras.R[0] * flip.diagonal().view(1, 3)).unsqueeze(0), gtn.view(-1, 3))
                gtnorms = gtn.norm(dim=1, keepdim=True)
                valid = (gtnorms > 0.0001)[..., 0]
                gtn = torch.where(valid.view(-1, 1), gtn / gtnorms.clamp(min=1e-12), gtn)
                if grad_d_p is not None:
                    J = grad_d_p               # the forward-mode Jacobian of the sweep above
                else:
                    ds = self.deformer(self.TmpPs, defconds, self.batch_inds, ratio=ratio)
                    J = utils.compute_Jacobian(self.TmpPs, ds, True, True)
                gtn = utils.mtv3(J, gtn.view(-1, 3))
                normal_loss = (gtn - nx).norm(2, dim=1) * weights
                normal_loss = _scatter_mean(normal_loss[valid], self.batch_inds[valid], N).mean()
                self.info['normal_loss'] = normal_loss.item()
                total_loss = total_loss + conf.get_float('normal_weight') * normal_loss
        shared.__exit__(None, None, None)
        if count_step:
            self.forward_time += 1
        return total_loss

    # ---- regularisers of forward(): network.py:552-593 ---------------------------------------------
    def _regularisers(self, eik_pts, base, N, d_cond, poses, trans, ratio, frame_ids):
        """offset loss (mean |translator offset| on the eikonal samples), def_regu (log-singular-value GM
        penalty on the translator Jacobian, singular values computed ON THE DEVICE: csrc/svals3x3.cu replaces
        the reference's CPU torch.svd round trip) and the DCT temporal loss on the posed skeleton."""
        conf = self.conf
        out = torch.zeros((), device=eik_pts.device)
        tr = self.deformer.defs[0] if hasattr(self.deformer, "defs") else None
        if conf is None or tr is None:
            return out
        if 'offset_weight' in conf and conf.get_float('offset_weight') >= 0.:
            w = conf.get_float('offset_weight')
            with torch.set_grad_enabled(w > 0.):
                off = self._offset(eik_pts.view(1, -1, 3).expand(N, -1, 3), d_cond, ratio)
                off = off.reshape(-1, 3).norm(p=2, dim=-1).mean()
            self.info['offset_loss'] = off.item()
            if w > 0.:
                out = out + off * w
        if 'def_regu' in conf and conf.get_float('def_regu.weight') > 0.:
            pts = torch.cat([base, utils.sample_points(base, 1.8, 0.01, 0)], dim=0).view(1, -1, 3).expand(N, -1, 3)
            pts = pts.detach().requires_grad_()
            if utils.train_fused(self.deformer):
                # translator Jacobian as a forward-mode output: J = I + d offset / d p
                n_, m_ = pts.shape[0], pts.shape[1]
                cr = d_cond.view(n_, 1, -1).expand(n_, m_, d_cond.shape[-1]).reshape(n_ * m_, -1)
                _, Joff = tr.forward_train(pts.reshape(-1, 3), cr, ratio, want_jac=True)
                J = torch.eye(3, device=pts.device).unsqueeze(0) + Joff
            else:
                dv = tr(pts, d_cond, ratio=ratio)
                J = utils.compute_Jacobian(pts, dv, True, True)
            sv = torch.log(utils.singular_values_3x3(J))
            dl = utils.GMRobustError((sv * sv).sum(1), conf.get_float('def_regu.c'), True).mean()
            self.info['def_loss'] = dl.item()
            out = out + dl * conf.get_float('def_regu.weight')
        if (poses.requires_grad or trans.requires_grad) and 'dct_weight' in conf and conf.get_float('dct_weight') > 0. \
                and hasattr(self, "dctnull"):
            klen, nlen = self.dctnull.shape
            bp, _ = self.dataset.get_batchframe_data('poses', frame_ids, nlen)
            bt, _ = self.dataset.get_batchframe_data('trans', frame_ids, nlen)
            pj = self.deformer.defs[1].posedSkeleton([bp.reshape(N * nlen, 24, 3), bt.reshape(N * nlen, 3)])
            dct = (self.dctnull[None, :, :, None] * pj.reshape(N, 1, nlen, 72)).sum(2).abs().mean()
            self.info['dct_loss'] = dct.item()
            out = out + dct * conf.get_float('dct_weight')
        return out

    # ---- seed of the ray set: network.py:485-505 / 317-345 -----------------------------------------
    def _mesh_seed(self, defTmpVs, TmpVs, Tmpfs):
        """Rasterise the deformed template and pick, per covered pixel, the front-most face hit and its
        canonical-space start point (utils.FindSurfacePs).  Uses the injected `raster_seed` callable when set
        (signature: (defTmpVs [N,V,3], TmpVs, Tmpfs, cameras) -> fragments-like or seed dict), else the
        pytorch3d mesh rasteriser held by maskRender."""
        N, V = defTmpVs.shape[0], TmpVs.shape[0]
        if self.raster_seed is not None:
            r = self.raster_seed(defTmpVs.detach(), TmpVs.detach(), Tmpfs, self.maskRender.rasterizer.cameras
                                 if self.maskRender is not None else None)
            if isinstance(r, dict):
                return r['batch_inds'], r['row_inds'], r['col_inds'], r['initTmpPs'], r.get('front_face_ids')
            return utils.FindSurfacePs(TmpVs.detach(), Tmpfs, r)
        from .raster import MeshRenderer, SilhouetteRenderer
        if isinstance(self.maskRender, SilhouetteRenderer):      # built-in device rasteriser (csrc/raster.cu)
            _, frags = self.maskRender(defTmpVs.detach(), Tmpfs)
            return utils.FindSurfacePs(TmpVs.detach(), Tmpfs, frags)
        if isinstance(self.maskRender, MeshRenderer):            # same rasteriser; the seed needs no shading
            frags = self.maskRender.rasterizer(defTmpVs.detach(), Tmpfs)
            return utils.FindSurfacePs(TmpVs.detach(), Tmpfs, frags)
        P = _p3d()
        meshes = P.Meshes(verts=[v.view(V, 3) for v in torch.split(defTmpVs.detach(), 1)], faces=[Tmpfs] * N)
        _, frags = self.maskRender(meshes)
        return utils.FindSurfacePs(TmpVs.detach(), Tmpfs, frags)

    def forward(self, datas, sample_pix, ratio, frame_ids, root=None, **kwargs):
        """One optimisation step's loss (network.py:451-644): remesh every `remesh_intersect` steps,
        deform the template, point-cloud silhouette loss with its inner SGD step on the template vertices
        (computeTmpPcLoss), then the ray losses (forward_rays)."""
        device = frame_ids.device
        gtMs = datas['mask'].to(device)
        N = frame_ids.numel()
        cameras, H, W = self._cameras(N, device)
        if self.maskRender is not None and hasattr(self.maskRender, "rasterizer"):
            self.maskRender.rasterizer.cameras = cameras
        if self.pcRender is not None:
            self.pcRender.rasterizer.cameras = cameras
        self.info = {}
        self.root = None
        if self.TmpVs is None or self.Tmpfs is None or self.forward_time % self.remesh_intersect == 0:
            self.update_hierarchical_config(device)
            self.TmpVs, self.Tmpfs = self.discretizeSDF(ratio, None, -self.sdfShrinkRadius)
            if self.TmpVs.shape[0] == 0:
                print('tmp sdf vanished...')
                assert False
            self.remesh_time = 1. + np.floor(self.remesh_time)
            self.TmpVs.requires_grad = True
            self.TmpOptimizer = torch.optim.SGD([self.TmpVs], lr=0.05, momentum=0.9)
            self.TmpVid, self.TmpFid = vertex_face_pairs(self.Tmpfs, self.TmpVs.shape[0])
            self.mesh_reg_topo = None
            self.root = root
        oldTmpVs = self.TmpVs.detach().clone() if self.root else None
        poses, trans, d_cond, _ = self.dataset.get_grad_parameters(frame_ids, device)
        defconds = [d_cond, [poses, trans]]
        defTmpVs = self._deform(self.TmpVs[None, :, :].expand(N, -1, 3), defconds, None, ratio)
        # the translator offset of this deform, for the snapshot's def1 meshes (later calls overwrite defs[0].offset)
        offset = self.deformer.defs[0].offset.detach().view(N, -1, 3) if self.root else None
        with torch.no_grad():
            bi, ri, ci, ps, _ = self._mesh_seed(defTmpVs, self.TmpVs, self.Tmpfs)
        pc_loss, masks, mgtMs = self._pc_silhouette_loss(defTmpVs, defconds, gtMs, H, W, ratio)
        if self.root:
            self.save_debug(oldTmpVs, self.Tmpfs, defTmpVs, offset, masks, gtMs, mgtMs, datas, bi, ri, ci, ps,
                            [d_cond.detach(), [poses.detach(), trans.detach()]], ratio, cameras)
        sel = gtMs[bi, ri, ci] > 0.      # colour losses only where render mask and gt mask intersect
        bi, ri, ci, ps = bi[sel], ri[sel], ci[sel], ps[sel]
        sample_pix = self.conf.get_int('sample_pix_num') if 'sample_pix_num' in self.conf else sample_pix
        if bi.shape[0] > sample_pix * N:
            sel = (torch.rand(bi.shape[0]) < float(sample_pix * N) / float(bi.shape[0])).to(device)
            bi, ri, ci, ps = bi[sel], ri[sel], ci[sel], ps[sel]
        TmpVnum = self.TmpVs.shape[0]
        extra = self.TmpVs[(torch.rand(TmpVnum) < 4096. / float(TmpVnum)).to(device)].detach()
        info_pc = self.info
        loss = pc_loss + self.forward_rays(datas, bi, ri, ci, ps, ratio, frame_ids, extra_points=extra,
                                           count_step=False)
        self.info.update({k: v for k, v in info_pc.items() if k not in self.info})
        self.remesh_time = np.floor(self.remesh_time) + float(self.forward_time % self.remesh_intersect) \
            / float(self.remesh_intersect)
        self.info['remesh'] = self.remesh_time
        self.forward_time += 1
        return loss

    def _pc_silhouette_loss(self, defTmpVs, defconds, gtMs, H, W, ratio):
        """network.py:497-507: soft point-cloud silhouette of the deformed template vs the (dilated) gt
        mask, then computeTmpPcLoss.  Without a point renderer (no level applied yet, none injected) the term is
        unavailable: that is an error unless `allow_missing_pc_loss` is set -- never a silent omission.
        -> (loss, point-cloud masks, dilated gt mask or None when the radius rounds to 0)."""
        self.info['pc_loss'] = {}
        if self.pcRender is None:
            if getattr(self, "allow_missing_pc_loss", False):
                self.info['pc_loss']['skipped'] = True
                return torch.zeros((), device=defTmpVs.device), None, None
            raise RuntimeError("OptimNetwork.forward: no point renderer (pcRender) -- install pytorch3d, inject one, "
                               "or set allow_missing_pc_loss=True to train without the silhouette term")
        N, V = defTmpVs.shape[0], self.TmpVs.shape[0]
        if getattr(self.pcRender, "takes_tensors", False):
            # a point renderer working on the [N,V,3] tensor directly (no pytorch3d containers)
            masks = self.pcRender(defTmpVs)
            radius = float(getattr(self.pcRender, "radius", 0.0))
            meshes = defTmpVs
        else:
            P = _p3d()
            meshes = P.Meshes(verts=[v.view(V, 3) for v in torch.split(defTmpVs, 1)], faces=[self.Tmpfs] * N)
            feats = [torch.ones(V, 1, device=defTmpVs.device) for _ in range(N)]
            masks, _ = self.pcRender(P.Pointclouds(points=meshes.verts_list(), features=feats))
            radius = self.pcRender.rasterizer.raster_settings.radius
        radius = int(np.round(radius / 2. * float(min(H, W)) / 1.2))
        mgtMs = None
        if radius > 0:
            mgtMs = torch.nn.functional.max_pool2d(gtMs, kernel_size=2 * radius + 1, stride=1, padding=radius)
        loss = self.computeTmpPcLoss(meshes, defconds, masks, gtMs if mgtMs is None else mgtMs, ratio)
        return loss, masks, mgtMs

    # ---- network.py:374-447 ---------------------------------------------------------------------
    def save_debug(self, TmpVs, Tmpfs, defTmpVs, offset, masks, gtMs, mgtMs, datas, batch_inds, row_inds, col_inds,
                   initTmpPs, defconds, ratio, cameras):
        """The progress snapshot of a remesh step, written under self.root: tmp.ply (the template before the inner
        SGD step), def_i.ply (deformed template of frame i), def1_i.ply (template + translator offset), m_i.png (point
        silhouette), mgm_i.png (dilated gt mask, when the radius is above 0) and, when self.draw is set, rgb_i.png /
        gtrgb_i.png / normal_i.png: the traced colour and the deformed-surface normal of every covered pixel.
        Builds no graph that outlives it, writes no .grad and draws no random numbers, so the step's loss and gradients do
        not depend on it."""
        if self.root is None:
            return
        import cv2
        from . import snapshot as S
        root = self.root
        os.makedirs(root, exist_ok=True)
        with torch.no_grad():
            S.write_ply(osp.join(root, 'tmp.ply'), TmpVs, Tmpfs)
            for ind in range(defTmpVs.shape[0]):
                S.write_ply(osp.join(root, 'def_%d.ply' % ind), defTmpVs[ind], Tmpfs)
            for ind in range(offset.shape[0]):
                S.write_ply(osp.join(root, 'def1_%d.ply' % ind), TmpVs + offset[ind], Tmpfs)
            if masks is not None:
                for ind, img in enumerate(S.mask_image(masks)):
                    cv2.imwrite(osp.join(root, 'm%d.png' % ind), img)
            if mgtMs is not None:
                for ind, img in enumerate(S.mask_image(mgtMs)):
                    cv2.imwrite(osp.join(root, 'mgm%d.png' % ind), img)
            if not self.draw:
                return
            gtCs = datas['img'].to(initTmpPs.device)
            print('draw %d points' % initTmpPs.shape[0])
            tcolors, tnormals = self._draw_rays(batch_inds, row_inds, col_inds, initTmpPs, cameras, defconds, ratio)
            colors = S.color_image(tcolors, batch_inds, row_inds, col_inds, gtCs)
            normals = S.normal_image(tnormals, batch_inds, row_inds, col_inds, gtCs)
            gtcolors = S.gt_color_image(gtCs)
            for ind in range(colors.shape[0]):
                cv2.imwrite(osp.join(root, 'rgb%d.png' % ind), colors[ind])
                cv2.imwrite(osp.join(root, 'gtrgb%d.png' % ind), gtcolors[ind])
                cv2.imwrite(osp.join(root, 'normal%d.png' % ind), normals[ind])
        self.draw = False

    def _draw_rays(self, batch_inds, row_inds, col_inds, initTmpPs, cameras, defconds, ratio, chunk=1 << 18):
        """Colour and camera-frame deformed normal of every seed pixel (network.py:405-424): trace as infer_rays does,
        then one shading pass per chunk that also returns the deformed normal.  The reference turns the normals of
        every frame by cameras.R[0]; so does this.  -> ([P,3] colours, [P,3] normals)"""
        pix = torch.cat([col_inds.view(-1, 1), row_inds.view(-1, 1), torch.ones_like(col_inds.view(-1, 1))], dim=-1)
        rays = cameras.view_rays(pix.float())
        cam_pos = cameras.cam_pos().detach()
        R0 = cameras.R[0].detach()
        tcolors, tnormals = [], []
        for rays_, ps_, bi_ in zip(torch.split(rays, chunk), torch.split(initTmpPs, chunk), torch.split(batch_inds, chunk)):
            with torch.enable_grad():
                # user-supplied field modules trace by autograd w.r.t. the points (FindSurfacePs._optimize_generic); the
                # fused tracer builds no graph either way.  Neither writes .grad.
                ps_, _ = utils.OptimizeSurfacePs(cam_pos, rays_.detach(), ps_.clone(), bi_, self.sdf, ratio,
                                                 self.deformer, defconds, dthreshold=1.e-4, athreshold=self.angThred,
                                                 w1=3.05, w2=1., times=30)
            ps_ = ps_.detach()
            if hasattr(self.sdf, "forward_fused"):
                _, _, rgb, nx = utils.shade_rays(self.sdf, self.deformer, self.netRender, ps_, rays_, defconds, bi_,
                                                 ratio, deformed_normals=True, cam_R0=R0)
            else:
                # user-supplied field modules: infer_rays' autograd sequence for the colour, then the deformed normal
                with torch.enable_grad():
                    ps_ = ps_.requires_grad_(True)
                    sdfs = self.sdf(ps_, ratio)
                    n0 = torch.autograd.grad(sdfs, ps_, torch.ones_like(sdfs))[0]
                    n0 = n0 / n0.norm(dim=1, keepdim=True)
                    crays, defVs = utils.compute_cardinal_rays(self.deformer, ps_, rays_, defconds, bi_, ratio, 'test')
                    nx, _ = utils.compute_deformed_normals(self.sdf, self.deformer, ps_, defconds, bi_, ratio, 'test')
                self.sdf(ps_, ratio)          # rendcond of these points, without a graph
                rgb = utils.compute_netRender_color(self.netRender, ps_, defVs, n0, crays, self.sdf.rendcond, None,
                                                    ratio)
                nx = utils.camera_normals(nx.detach(), R0)
            tcolors.append(rgb)
            tnormals.append(nx)
        return torch.cat(tcolors, dim=0), torch.cat(tnormals, dim=0)

    # ---- network.py:647-697 ---------------------------------------------------------------------
    def computeTmpPcLoss(self, defMeshes, defconds, imgs, gtMs, ratio):
        """IoU silhouette loss + template mesh regularisers, ONE inner SGD step on the template vertices,
        then |f(TmpVs)| which ties the SDF to the moved template (returned to the outer optimiser)."""
        conf = self.conf
        N = gtMs.shape[0]
        masks = imgs[..., -1]
        inter = (masks * gtMs).view(N, -1).sum(1)
        union = (masks + gtMs - masks * gtMs).abs().view(N, -1).sum(1)
        mask_loss = (1. - inter / union).mean()
        self.info['pc_loss']['mask_loss'] = mask_loss.item()
        loss = mask_loss * (conf.get_float('pc_weight.mask_weight') if 'pc_weight.mask_weight' in conf else 1.)
        has_pc = 'pc_weight' in conf
        tmpMesh = regs = None
        for i, (key, tag, fn) in enumerate((
                ('laplacian_weight', 'lap_loss', lambda P, m: P.mesh_laplacian_smoothing(m, method='uniform')),
                ('edge_weight', 'edge_loss', lambda P, m: P.mesh_edge_loss(m, target_length=0.)),
                ('norm_weight', 'norm_loss', lambda P, m: P.mesh_normal_consistency(m)))):
            w = conf.get_float('pc_weight.' + key) if (has_pc and ('pc_weight.' + key) in conf) else -1.
            if w <= 0.:
                continue
            if torch.is_tensor(defMeshes):
                # the silhouette ran on tensors: all three terms from one device evaluation (csrc/mesh_reg.cu)
                if regs is None:
                    if self.mesh_reg_topo is None:
                        self.mesh_reg_topo = ops.mesh_reg_topology(self.Tmpfs, self.TmpVs.shape[0])
                    regs = ops.mesh_regularizers(self.TmpVs, self.mesh_reg_topo)
                term = w * regs[i]
            else:
                P = _p3d()      # pytorch3d's mesh regularisers on its own containers
                if tmpMesh is None:
                    tmpMesh = P.Meshes(verts=[self.TmpVs], faces=[self.Tmpfs])
                term = w * fn(P, tmpMesh)
            loss = loss + term
            self.info['pc_loss'][tag] = term.item() / w
        cw = conf.get_float('pc_weight.def_consistent.weight') if 'pc_weight.def_consistent' in conf else -1.
        if cw > 0.:
            rigid = self.deformer.defs[1](self.TmpVs.view(1, -1, 3).expand(N, -1, 3), defconds[1])
            dv = defMeshes if torch.is_tensor(defMeshes) else defMeshes.verts_padded()
            d2 = ((dv - rigid) ** 2).sum(-1)
            c = conf.get_float('pc_weight.def_consistent.c')
            cl = utils.GMRobustError(d2, c, True).mean() if c > 0. else torch.sqrt(d2).mean()
            self.info['pc_loss']['defconst_loss'] = cl.item()
            loss = loss + cl * cw
        self.TmpOptimizer.zero_grad()
        loss.backward()
        self.TmpOptimizer.step()
        pred = self._sdf_value(self.TmpVs, ratio).view(-1) + self.sdfShrinkRadius
        if utils.train_fused(self.deformer, self.sdf):
            # d|x|/dx = sign(x) is a DECISION on values that sit on the zero set by construction (template vertices):
            # it is taken on the fp32 engine's value (tensor-core values inside their error band are re-evaluated,
            # ops.sdf_refine_band), then applied to the differentiable tensor-core evaluation
            with torch.no_grad():
                f32 = self.sdf.forward_fused(self.TmpVs.detach(), ratio, False, False,
                                             refine_about=-self.sdfShrinkRadius)[0].view(-1) + self.sdfShrinkRadius
            sdf_loss = (torch.sign(f32) * pred).mean()
        else:
            sdf_loss = pred.abs().mean()
        self.info['pc_loss_sdf'] = sdf_loss.item()
        return sdf_loss * (conf.get_float('pc_weight.weight') if has_pc else 60.)

    # ---- network.py:306-372 ---------------------------------------------------------------------
    def infer(self, TmpVs, Tmpfs, H, W, ratio, frame_ids, notcolor=False, gts=None):
        """Renders N frames: shaded images of the deformed and of the translator-only template (whatever shader
        maskRender holds), then the neural colour of every covered pixel through infer_rays.
        -> (colors uint8 [N,H,W,3] | None, imgs, def1imgs, deformed vertices).
        With a built-in renderer (raster.SilhouetteRenderer / raster.MeshRenderer) no pytorch3d is needed."""
        from .raster import MeshRenderer, SilhouetteRenderer
        if isinstance(self.maskRender, (SilhouetteRenderer, MeshRenderer)):
            return self._infer_builtin(TmpVs, Tmpfs, ratio, frame_ids, notcolor, gts)
        device = TmpVs.device
        P = _p3d()
        N, V = frame_ids.numel(), TmpVs.shape[0]
        with torch.no_grad():
            cameras, H, W = self._cameras(N, device)
            self.maskRender.rasterizer.cameras = cameras
            if self.pcRender is not None:
                self.pcRender.rasterizer.cameras = cameras
            poses, trans, d_cond, _ = self.dataset.get_grad_parameters(frame_ids, device)
            tex = lambda: P.TexturesVertex([torch.ones_like(TmpVs) for _ in range(N)])
            defTmpVs = self.deformer(TmpVs[None].expand(N, -1, 3), [d_cond, [poses, trans]], ratio=ratio)
            meshes = P.Meshes(verts=[v.view(V, 3) for v in torch.split(defTmpVs, 1)], faces=[Tmpfs] * N, textures=tex())
            defMeshVs = defTmpVs.detach().cpu().numpy()
            imgs, frags = self.maskRender(meshes)
            masks = None
            if gts:
                m = (frags.pix_to_face >= 0).float()[..., 0]
                g = gts['mask']
                gts['maskE'] = (1. - (m * g).view(N, -1).sum(1) / (m + g - m * g).abs().view(N, -1).sum(1)).cpu().numpy()
                masks = m > 0.
                imgs = imgs[..., :3]
                if 'image' in gts:
                    imgs[~masks] = gts['image'][~masks][:, [2, 1, 0]]
            imgs = torch.clamp(imgs * 255., min=0., max=255.).cpu().numpy().astype(np.uint8)
            d1 = self.deformer.defs[0](TmpVs[None].expand(N, -1, 3), d_cond, ratio=ratio)
            meshes1 = P.Meshes(verts=[v.view(V, 3) for v in torch.split(d1, 1)], faces=[Tmpfs] * N, textures=tex())
            newTs = self.dataset.trans.mean(0).to(device)[None, :]
            front = torch.tensor([[[-1., 0., 0.], [0., 1., 0.], [0., 0., -1.]]], device=device).repeat(N, 1, 1)
            focals, pps, _, _, _, _ = self.dataset.get_camera_parameters(N, device)
            cam1 = type(cameras)(focals, pps, front, newTs.repeat(N, 1), image_size=[(W, H)]).to(device)
            def1imgs, _ = self.maskRender(meshes1, cameras=cam1,
                                          lights=P.PointLights(device=device, location=((0, 1, newTs[0, 2].item()),)))
            def1imgs = torch.clamp(def1imgs * 255., min=0., max=255.).cpu().numpy().astype(np.uint8)
            bi, ri, ci, ps, _ = utils.FindSurfacePs(TmpVs.detach(), Tmpfs, frags)
        if notcolor:
            return None, imgs, def1imgs, defMeshVs
        print('draw %d points' % bi.shape[0])
        colors = self.infer_rays(bi, ri, ci, ps, H, W, ratio, frame_ids)
        if gts and 'image' in gts and masks is not None:
            colors[~masks] = gts['image'][~masks][:, :3] * 255.
        return colors.cpu().numpy().astype(np.uint8), imgs, def1imgs, defMeshVs

    def _infer_builtin(self, TmpVs, Tmpfs, ratio, frame_ids, notcolor, gts):
        """infer() on the built-in renderer: the same sequence (network.py:306-372) with the device rasteriser and,
        for a MeshRenderer, the device Phong shader (csrc/mesh_shade.cu) in place of pytorch3d's Meshes pipeline."""
        from .raster import PointLights
        device = TmpVs.device
        N = frame_ids.numel()
        with torch.no_grad():
            cameras, H, W = self._cameras(N, device)
            self.maskRender.rasterizer.cameras = cameras
            if self.pcRender is not None:
                self.pcRender.rasterizer.cameras = cameras
            poses, trans, d_cond, _ = self.dataset.get_grad_parameters(frame_ids, device)
            defTmpVs = self.deformer(TmpVs[None].expand(N, -1, 3), [d_cond, [poses, trans]], ratio=ratio)
            defMeshVs = defTmpVs.detach().cpu().numpy()
            imgs, frags = self.maskRender(defTmpVs.detach(), Tmpfs)
            masks = None
            if gts:
                m = (frags.pix_to_face >= 0).float()[..., 0]
                g = gts['mask']
                gts['maskE'] = (1. - (m * g).view(N, -1).sum(1) / (m + g - m * g).abs().view(N, -1).sum(1)).cpu().numpy()
                masks = m > 0.
                imgs = imgs[..., :3]
                if 'image' in gts:
                    imgs[~masks] = gts['image'][~masks][:, [2, 1, 0]]
            imgs = torch.clamp(imgs * 255., min=0., max=255.).cpu().numpy().astype(np.uint8)
            d1 = self.deformer.defs[0](TmpVs[None].expand(N, -1, 3), d_cond, ratio=ratio)
            newTs = self.dataset.trans.mean(0).to(device)[None, :]
            front = torch.tensor([[[-1., 0., 0.], [0., 1., 0.], [0., 0., -1.]]], device=device).repeat(N, 1, 1)
            focals, pps, _, _, _, _ = self.dataset.get_camera_parameters(N, device)
            cam1 = type(cameras)(focals, pps, front, newTs.repeat(N, 1), image_size=[(W, H)]).to(device)
            def1imgs, _ = self.maskRender(d1.detach(), Tmpfs, cameras=cam1,
                                          lights=PointLights(device=device, location=((0, 1, newTs[0, 2].item()),)))
            def1imgs = torch.clamp(def1imgs * 255., min=0., max=255.).cpu().numpy().astype(np.uint8)
            bi, ri, ci, ps, _ = utils.FindSurfacePs(TmpVs.detach(), Tmpfs, frags)
        if notcolor:
            return None, imgs, def1imgs, defMeshVs
        print('draw %d points' % bi.shape[0])
        colors = self.infer_rays(bi, ri, ci, ps, H, W, ratio, frame_ids)
        if gts and 'image' in gts and masks is not None:
            colors[~masks] = gts['image'][~masks][:, :3] * 255.
        return colors.cpu().numpy().astype(np.uint8), imgs, def1imgs, defMeshVs

    # ---- network.py:702-814 ---------------------------------------------------------------------
    def propagateTmpPsGrad(self, frame_ids, ratio):
        if self.TmpPs is None or self.TmpPs.grad is None:
            self.info['invInfo'] = (-1, -1)
            return
        device = self.TmpPs.device
        poses, trans, d_cond, _ = self.dataset.get_grad_parameters(frame_ids, device)
        defconds = [d_cond, [poses, trans]]
        cameras, _, _ = self._cameras(frame_ids.numel(), device)
        grad_l_p = self.TmpPs.grad
        if self.rays.requires_grad:
            pix = torch.cat([self.col_inds.view(-1, 1), self.row_inds.view(-1, 1),
                             torch.ones_like(self.col_inds.view(-1, 1))], dim=-1)
            v = cameras.view_rays(pix.float())
        else:
            v = self.rays.detach()
        c = cameras.cam_pos()
        p = self.TmpPs
        fusable = hasattr(self.sdf, "forward_fused") and hasattr(self.deformer, "forward_fused") \
            and self.deformer._fusable()
        geom = getattr(self, "_tmp_geom", None)
        if geom is not None and geom[0] is p:
            grad_f_p, grad_d_p = geom[1], geom[2]        # evaluated at exactly these points by forward_rays
        elif fusable:
            # grad f and dD/dp at p from the fused forward-mode kernels: no graph, no 1+3 VJP passes
            with torch.no_grad():
                _, grad_f_p, _ = self.sdf.forward_fused(p.detach(), ratio, want_grad=True, want_feat=False)
                _, grad_d_p, _ = self.deformer.forward_fused(p.detach(), [c_.detach() if torch.is_tensor(c_) else
                                                                          [t.detach() for t in c_] for c_ in defconds],
                                                             self.batch_inds, ratio, want_jac=True)
        else:
            f = self.sdf(p, ratio)
            grad_f_p = torch.autograd.grad(f, p, torch.ones_like(f), retain_graph=False)[0]
            d = self.deformer(p, defconds, self.batch_inds, ratio=ratio)
            grad_d_p = utils.compute_Jacobian(p, d, False, False)
        v_cross = _cross_matrix(v.detach())
        a1 = (v_cross.unsqueeze(-1) * grad_d_p.unsqueeze(-3)).sum(-2)          # [v]x J, elementwise (no GEMM launch)
        b = torch.cat([grad_f_p.view(-1, 1, 3), a1], dim=1)           # [P,4,3]
        btb = (b.unsqueeze(-1) * b.unsqueeze(-2)).sum(1)
        btb_inv, check = Fast3x3Minv(btb.contiguous())
        self.info['invInfo'] = (check.numel(), check.sum().item())
        # rhs = dL/dp (b^T b)^-1 b^T   [P,1,4]
        rhs_1 = utils.mv3(b, utils.mtv3(btb_inv, grad_l_p.view(-1, 3))).view(-1, 1, 4)
        loss = 0.
        # theta: VJP of the sdf with cotangent -rhs[...,0]
        train_fused = fusable and utils.train_fused(self.deformer, self.sdf)
        params = [q for q in self.sdf.parameters() if q.requires_grad]
        if train_fused:   # first-order VJP through the tensor-core training engine (value rows only, no feature head)
            f_p = self.sdf.forward_train(p.detach(), ratio, want_grad=False, want_feat=False)[0]
        else:
            f_p = self.sdf(p, ratio)
        grads = torch.autograd.grad(f_p, params, -rhs_1[:, :, 0], allow_unused=True)
        grads = [g if g is not None else torch.zeros_like(q) for g, q in zip(grads, params)]
        for q, g in zip(params, grads):
            loss = loss + (q * g).sum()
        # phi, latent codes, pose: VJP of the deformer with cotangent rhs[...,1:] (-[v]x)
        opt_defconds = []
        for dc in defconds:
            for t in (dc if isinstance(dc, list) else [dc]):
                if t.requires_grad:
                    opt_defconds.append(t)
        params = [q for q in self.deformer.parameters() if q.requires_grad]
        if train_fused:
            d = self.deformer.forward_train(p.detach(), defconds, self.batch_inds, ratio, want_jac=False)[0]
        else:
            d = self.deformer(p, defconds, self.batch_inds, ratio=ratio)
        temp = utils.mtv3(-v_cross, rhs_1[:, 0, -3:])
        grads = torch.autograd.grad(d, params + opt_defconds, temp)
        for q, g in zip(params + opt_defconds, grads):
            loss = loss + (q * g).sum()
        if v.requires_grad:
            dc_cross = _cross_matrix(d.detach() - c.detach().view(1, 3))
            loss = loss + (v * utils.mtv3(dc_cross, rhs_1[:, 0, -3:])).sum()
        if c.requires_grad:
            loss = loss + (c * (-temp.sum(0))).sum()
        loss.backward()


# ---- network.py:828-909 -------------------------------------------------------------------------
def getOptNet(dataset, N, bmins, bmaxs, resolutions, device, conf, use_initial_sdf=True, use_initial_skinner=True):
    """Builds the OptimNetwork of a sequence: SDF (optionally from `initial_sdf_idr_*.pth`), LBS field
    (from `initial_skinner_*.pth` or computed from SMPL and cached there), translator, rendering network,
    cameras, coarse-to-fine MC engine and the silhouette renderer.  -> (optNet, sdf_initialized), where
    sdf_initialized > 0 asks the caller to run initializeTmpSDF for that many epochs."""
    from MCAcc import Seg3dLossless
    from . import RenderNet
    from .network import getTmpSdf
    from .Deformer import initialLBSkinner, getTranslatorNet, CompositeDeformer, LBSkinner
    sdf_multires = conf.get_int('sdf_net.multires')
    condlen = conf.get_int('render_net.condlen')
    tmpSdf = getTmpSdf(device, sdf_multires, 0.6, condlen)
    sdf_initialized = conf.get_int('train.initial_iters')
    pose_type = conf.get_int('train.skinner_pose_type') if 'train.skinner_pose_type' in conf else 0
    sdf_file = osp.join(dataset.root, 'initial_sdf_idr_%d_%d.pth' % (sdf_multires, pose_type))
    if osp.isfile(sdf_file) and use_initial_sdf:
        tmpSdf.load_state_dict(torch.load(sdf_file, map_location='cpu'))
        sdf_initialized = -1
    elif sdf_initialized <= 0:
        sdf_initialized = 1200
    skinner_file = osp.join(dataset.root, 'initial_skinner_%d.pth' % pose_type)
    if osp.isfile(skinner_file) and use_initial_skinner:
        d = torch.load(skinner_file, map_location='cpu', weights_only=False)
        skinner = LBSkinner(d['ws'], d['bmins'], d['bmaxs'], d['Js'], d['parents'], init_pose=d['init_pose'],
                            align_corners=False)
        tmpBodyVs, tmpBodyFs = d['tmpBodyVs'], d['tmpBodyFs']
    else:
        # A pose as the rest pose keeps the weight volume's box small
        initPose = torch.from_numpy(utils.smpl_tmp_Apose(pose_type)).view(1, 24, 3).to(device)
        skinner, tmpBodyVs, tmpBodyFs = initialLBSkinner(dataset.gender, dataset.shape.to(device), initPose,
                                                         (128 + 1, 224 + 1, 64 + 1), bmins, bmaxs)
        torch.save({'ws': skinner.ws, 'bmins': skinner.b_min, 'bmaxs': skinner.b_max, 'Js': skinner.Js,
                    'parents': skinner.parents, 'init_pose': skinner.init_pose, 'tmpBodyVs': tmpBodyVs,
                    'tmpBodyFs': tmpBodyFs}, skinner_file)
    deformer = CompositeDeformer([getTranslatorNet(device, conf.get_config('mlp_deformer')), skinner]).to(device)
    cam = dataset.camera_params
    cameras = RectifiedPerspectiveCameras(cam['focal_length'].view(1, 2).expand(N, 2),
                                          cam['princeple_points'].view(1, 2).expand(N, 2),
                                          utils.quat2mat(cam['cam2world_coord_quat'].view(1, 4)).expand(N, 3, 3),
                                          cam['world2cam_coord_trans'].view(1, 3).expand(N, 3),
                                          image_size=[(dataset.W, dataset.H)]).to(device)
    engine = Seg3dLossless(query_func=None, b_min=skinner.b_min.tolist(), b_max=skinner.b_max.tolist(),
                           resolutions=resolutions, align_corners=False, balance_value=0.0, device=device,
                           visualize=False, debug=False, use_cuda_impl=False, faster=False)
    renderer = _silhouette_renderer(cameras, dataset.H, dataset.W)
    rendnet = RenderNet.getRenderNet(device, conf.get_config('render_net'))
    optNet = OptimNetwork(tmpSdf, deformer, engine, renderer, rendnet, conf=conf.get_config('loss_coarse'))
    optNet.remesh_intersect = conf.get_int('train.coarse.point_render.remesh_intersect')
    tmpBodyVs = torch.as_tensor(tmpBodyVs).float()
    tmpBodyFs = torch.as_tensor(tmpBodyFs).long()
    optNet.register_buffer('tmpBodyVs', tmpBodyVs)
    optNet.register_buffer('tmpBodyFs', tmpBodyFs)
    # vertex normals of the body template: normalised sum of the incident unit face normals (what openmesh's
    # update_normals computes, network.py:899-903), from one sort of the face table instead of a half-edge mesh
    vid, fid = vertex_face_pairs(tmpBodyFs, tmpBodyVs.shape[0])
    optNet.register_buffer('tmpBodyNs', utils.compute_vnorms(tmpBodyVs, tmpBodyFs, vid, fid))
    optNet = optNet.to(device)
    optNet.dataset = dataset
    dataset.store_device = device       # the loader keeps the sequence's frames on this device (dataset.frame_store)
    if dataset.poses.requires_grad or dataset.trans.requires_grad:
        optNet.dctnull = utils.DCTNullSpace(10, 30).to(device)
    return optNet, sdf_initialized


def _silhouette_renderer(cameras, H, W):
    try:
        P = _p3d()
    except RuntimeError:
        # no pytorch3d: the built-in device rasteriser provides the fragments the ray seed needs
        from .raster import MeshRasterizer, RasterSettings, SilhouetteRenderer
        return SilhouetteRenderer(MeshRasterizer(cameras, RasterSettings((H, W))))
    settings = P.RasterizationSettings(image_size=(H, W), blur_radius=0.,
                                       bin_size=int(2 ** max(np.ceil(np.log2(max(H, W))) - 4, 4)),
                                       faces_per_pixel=1, perspective_correct=True, clip_barycentric_coords=False,
                                       cull_backfaces=False)
    return P.MeshRendererWithFragments(rasterizer=P.MeshRasterizer(cameras=cameras, raster_settings=settings),
                                       shader=P.SoftSilhouetteShader())
