"""The training step's debug snapshot (OptimNetwork.save_debug, model/network.py:374-447) and the deformed normals of
the tensor-core shading pass it draws with (sr_tc_shade_point_deformed).

  * the entry point against a float64 restatement built from its own fp32 inputs, with singular J rows (fallback) and
    the camera rotation; its other outputs bit-identical to sr_tc_shade_point;
  * on traced points of the synthetic scene, the deformed normals against float64 on the kernel's own inputs, and
    against compute_deformed_normals on the FFMA engine wherever J is formed by the same decisions;
  * forward(..., root) without pytorch3d / trimesh: the reference's file set, each file against what the step computed;
  * the snapshot has no effect on the step: loss, info, gradients, template and RNG states bit-identical;
  * a draw with a user-supplied SDF (the autograd trace and shading) completes the step."""
import ctypes as C
import os
import sys

import cv2
import numpy as np
import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS32 = float(np.finfo(np.float32).eps)
FLIP = np.diag([-1., 1., -1.])
# Deformed normals of the tensor-core shading pass against compute_deformed_normals on the FFMA engine.  The template
# normals keep their documented band (test_gpu_narrow_shade.NORMAL_BAR); the deformed normal, J^-T applied to them,
# is held to the cardinal-ray band of the shading stage (test_gpu_parity.FP_TOL) on every point whose J is formed by
# the same decisions in both engines.  Two decisions make J piecewise: the translator's ReLUs (d offset / dp changes
# by a rank-one term when a hidden pre-activation changes sign) and the skinning cell of p + offset (the trilinear
# weights' gradient jumps across cell faces).  A point is decision-sensitive when a float64 evaluation of the
# translator puts a hidden pre-activation within RELU_MARGIN of zero, or when the two engines' p + offset land in
# different cells.  Measured on H100: every point outside the band (18 of 10 408, up to 1.8e-3) has a pre-activation
# within 1.0e-6 of zero, none changes cell, and its template normal is within 1.5e-5 of the FFMA one.
NORMAL_BAR = 5e-5
DEFN_BAND = 1e-4
RELU_MARGIN = 2e-6


# ---------------------------------------------------------------------------------------------------------------------
# the entry point against float64
# ---------------------------------------------------------------------------------------------------------------------
def _rotation(g):
    q, _ = np.linalg.qr(g.standard_normal((3, 3)))
    return q * np.sign(np.linalg.det(q))


def _inputs(P, seed):
    """pts, rays, grad, off4 (offset row + 3 tangent rows per point) with J = I + d offset / dp; the first 8 rows
    hold hand-built singular J (exact in fp32) and near-singular ones (|det| ~ 5e-5 < 1e-4)."""
    g = np.random.default_rng(seed)
    pts = g.uniform(-0.8, 0.8, (P, 3)).astype(np.float32)
    rays = g.standard_normal((P, 3))
    rays = (rays / np.linalg.norm(rays, axis=1, keepdims=True)).astype(np.float32)
    grad = (g.standard_normal((P, 3)) * g.uniform(0.5, 2.0, (P, 1))).astype(np.float32)
    J = np.eye(3)[None] + g.standard_normal((P, 3, 3)) * np.where(np.arange(P) % 3 == 0, 0.6, 0.15)[:, None, None]
    bad = np.abs(np.linalg.det(J)) < 0.05                                  # keep random rows clear of the threshold
    J[bad] = np.eye(3)[None] + g.standard_normal((int(bad.sum()), 3, 3)) * 0.05
    sing = [np.array([[1., 2., 3.], [2., 4., 6.], [.5, 1., .25]]),            # rank 2, det exactly 0
            np.array([[0., 0., 0.], [1., 2., 0.], [0., 1., 1.]]),             # zero row
            np.diag([1., 1., 5e-5]), np.diag([2., 1e-2, 2.5e-3]),            # |det| 5e-5
            np.array([[1., 1., 0.], [1., 1., 0.], [0., 0., 3.]]),
            np.diag([3., 3., 0.]), np.array([[1., 0., 0.], [0., 0., 1.], [0., 0., 1.]]), np.diag([1e-2, 1e-2, 0.5])]
    for i, s in enumerate(sing):
        J[i] = s
    off4 = np.zeros((P, 4, 3), np.float32)
    off4[:, 0] = g.uniform(-0.05, 0.05, (P, 3))
    off4[:, 1:] = np.transpose(J - np.eye(3)[None], (0, 2, 1))             # off4[4i+1+c][m] = Joff[m][c]
    return pts, rays, grad, off4.reshape(P * 4, 3), len(sing)


def _kernel_J(off4):
    """J exactly as the kernel forms it with M = I: Q = fl32(delta + Joff), then I Q = Q."""
    P = off4.shape[0] // 4
    Joff = np.transpose(off4.reshape(P, 4, 3)[:, 1:], (0, 2, 1))
    return (np.eye(3, dtype=np.float32)[None] + Joff).astype(np.float64)


def _launch(lib, ops, tens, deformed, R0=None):
    pts, rays, grad, off4 = tens
    P = pts.shape[0]
    out = [torch.full((P, 3), float("nan"), device=DEV) for _ in range(3)] + [torch.full((P,), 7, dtype=torch.uint8,
                                                                                         device=DEV)]
    if deformed:
        defn = torch.full((P, 3), float("nan"), device=DEV)
        r = None if R0 is None else (C.c_float * 9)(*[float(x) for x in np.asarray(R0, np.float32).reshape(9)])
        code = lib.sr_tc_shade_point_deformed(P, ops._p(pts), ops._p(rays), None, ops._p(grad), ops._p(off4), None,
                                              *[ops._p(t) for t in out], ops._p(defn), r, ops._stream())
        out.append(defn)
    else:
        code = lib.sr_tc_shade_point(P, ops._p(pts), ops._p(rays), None, ops._p(grad), ops._p(off4), None,
                                     *[ops._p(t) for t in out], ops._stream())
    assert code == 0
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("P", [600, 5000])
def test_entry_point_vs_float64(P):
    from selfreconcode_b200 import _lib, ops
    lib = _lib.load()
    assert (P < ops.TC_MIN_POINTS) == (P == 600)
    pts, rays, grad, off4, nsing = _inputs(P, seed=P)
    tens = [torch.from_numpy(a).to(DEV) for a in (pts, rays, grad, off4)]
    base = _launch(lib, ops, tens, False)
    R0 = _rotation(np.random.default_rng(P + 1))
    for rot in (None, R0):
        got = _launch(lib, ops, tens, True, rot)
        for a, b, name in zip(base, got[:4], ("normals", "crays", "dpos", "ok")):
            assert torch.equal(a, b), name                  # the shared outputs: same bits as sr_tc_shade_point
        ok = got[3].cpu().numpy().astype(bool)
        n = got[4].cpu().numpy().astype(np.float64)
        J = _kernel_J(off4)
        g = grad.astype(np.float64)
        det = np.linalg.det(J)
        assert not ok[:nsing].any(), "hand-built singular rows must take the fallback"
        assert ok[nsing:].all() and np.abs(det[nsing:]).min() > 1e-2
        # float64 restatement: normalize(J^-T g), fallback normalize(J g), on the kernel's decisions
        y = np.empty((P, 3))
        y[ok] = np.einsum('pkr,pk->pr', np.linalg.inv(J[ok]), g[ok])
        y[~ok] = np.einsum('prk,pk->pr', J[~ok], g[~ok])
        n64 = y / np.linalg.norm(y, axis=1, keepdims=True)
        # bound per row: the inverse applied to g has forward error ~ eps kappa(J) ||J^-1|| ||g|| (cofactors + det),
        # i.e. relative eps kappa(J) amp with amp = ||J^-T|| ||g|| / ||J^-T g||; the fallback's product eps ||J|| ||g||
        # / ||J g||; 32 eps covers the constants, the normalisation and (with rot) the rotation's 3-term sums
        sv = np.linalg.svd(J, compute_uv=False)
        kappa = sv[:, 0] / np.maximum(sv[:, 2], 1e-300)
        gn, yn = np.linalg.norm(g, axis=1), np.linalg.norm(y, axis=1)
        amp = np.where(ok, gn / np.maximum(sv[:, 2], 1e-300) / yn, sv[:, 0] * gn / yn)
        bound = 32 * EPS32 * (np.where(ok, kappa, 1.0) * amp + 1.0)
        if rot is not None:
            n64 = n64 @ (FLIP @ rot.T).T
        err = np.abs(n - n64).max(1)
        well = ok & (kappa < 1e3)
        print("P=%d rot=%s: well-conditioned rows %d (kappa max %.1f), max |dn| %.2e, max |dn|/bound %.3f; "
              "fallback rows %d, max |dn| %.2e" % (P, rot is not None, well.sum(), kappa[well].max(), err[well].max(),
                                                    (err / bound)[well].max(), (~ok).sum(), err[~ok].max()))
        assert well.sum() > 0.9 * P
        assert np.all(err[well] <= bound[well])
        assert np.all(err[~ok] <= bound[~ok])
        assert np.isfinite(n).all()


def test_entry_point_rejects_missing_output():
    from selfreconcode_b200 import _lib, ops
    lib = _lib.load()
    pts, rays, grad, off4, _ = _inputs(64, seed=1)
    t = [torch.from_numpy(a).to(DEV) for a in (pts, rays, grad, off4)]
    out = [torch.empty(64, 3, device=DEV) for _ in range(3)] + [torch.empty(64, dtype=torch.uint8, device=DEV)]
    assert lib.sr_tc_shade_point_deformed(64, ops._p(t[0]), ops._p(t[1]), None, ops._p(t[2]), ops._p(t[3]), None,
                                          *[ops._p(x) for x in out], None, None, ops._stream()) == _lib.SR_EINVAL


# ---------------------------------------------------------------------------------------------------------------------
# the synthetic scene
# ---------------------------------------------------------------------------------------------------------------------
def _net(Hh=128, Ww=128, n_frames=3):
    """The scene and level set-up of test_gpu_points_silhouette._step, without running the step."""
    import utils
    from selfreconcode_b200 import synth
    from test_gpu_mesh_shade import _scene
    net, data, cams, _, _, fids = _scene(Hh, Ww, n_frames)
    conf = synth.reference_config()
    conf._find('train.coarse.point_render')['radius'] = 0.02
    for lvl in ('loss_coarse', 'loss_medium', 'loss_fine'):
        conf[lvl] = dict(conf[lvl], pc_weight=dict(weight=60., mask_weight=1., laplacian_weight=-10.,
                                                   edge_weight=-10., norm_weight=-0.001,
                                                   def_consistent=dict(weight=0.1, c=0.005)))
    loader = torch.utils.data.DataLoader(list(range(n_frames)), n_frames)
    net, loader = utils.set_hierarchical_config(conf, 'coarse', net, loader, synth.MC_LADDER_65)
    net.update_hierarchical_config(torch.device(DEV))
    return net, data, fids


def _datas(N, Hh, Ww):
    from test_gpu_mesh_shade import _gts
    g = torch.Generator().manual_seed(21)
    return {'img': (torch.rand(N, Hh, Ww, 3, generator=g) * 2 - 1).to(DEV), 'mask': _gts(N, Hh, Ww, image=False)['mask']}


def _traced(net, fids):
    """Seed pixels of the deformed template and their traced surface points, as save_debug's draw traces them."""
    import utils
    N = fids.numel()
    TmpVs, Tmpfs = net.discretizeSDF(H.RATIO, None, 0.0)
    cams, _, _ = net._cameras(N, DEV)
    net.maskRender.rasterizer.cameras = cams
    poses, trans, d_cond, _ = net.dataset.get_grad_parameters(fids, DEV)
    defconds = [d_cond.detach(), [poses.detach(), trans.detach()]]
    with torch.no_grad():
        defTmpVs = net.deformer(TmpVs.detach()[None].expand(N, -1, 3), defconds, ratio=H.RATIO)
        bi, ri, ci, ps, _ = net._mesh_seed(defTmpVs, TmpVs.detach(), Tmpfs)
        pix = torch.cat([ci.view(-1, 1), ri.view(-1, 1), torch.ones_like(ci.view(-1, 1))], dim=-1)
        rays = cams.view_rays(pix.float())
        pts, conv = utils.OptimizeSurfacePs(cams.cam_pos().detach(), rays, ps.clone(), bi, net.sdf, H.RATIO,
                                            net.deformer, defconds, dthreshold=1.e-4, athreshold=net.angThred,
                                            w1=3.05, w2=1., times=30)
    return pts, rays, bi, defconds, cams


def _lbs_matrices(net, pp, bi, defconds):
    """M = dD/dp' of the skinning at p' = pp [P,3], from the FFMA engine's lbs_point: the stock translator with a zero
    output layer has offset 0 and d offset / dp 0, so its J is M exactly."""
    from model.Deformer import MLPTranslator
    from selfreconcode_b200 import ops
    tr, sk = net.deformer.defs[0], net.deformer.defs[1]
    z = MLPTranslator(tr.feature_vector_size, tr.multires).to(pp.device)
    z.load_state_dict(tr.state_dict())
    last = getattr(z, "lin%d" % (z.num_layers - 2))
    with torch.no_grad():
        last.weight.zero_()
        last.bias.zero_()
    poses, trans = defconds[1]
    lbs = sk.lbs_state()
    lbs.set_pose(poses.view(poses.shape[0], 24, 3), trans)
    _, off, M, _ = ops.deform_forward(z.fused(H.RATIO), lbs, pp, bi, defconds[0], want_jac=True, want_offset=True)
    assert torch.all(off == 0)
    return M


def _kernel_inputs(net, pts, bi, defconds):
    """grad f and the translator's 4-row block as shade_and_render_tc computes them, and M at p + offset."""
    from selfreconcode_b200 import _lib, ops
    P = pts.shape[0]
    p = pts.detach().contiguous().float()
    bi64 = bi.contiguous().to(torch.int64)
    full = net.sdf.fused()
    full.set_pe_weights(net.sdf._pe_weights(H.RATIO['sdfRatio']))
    with torch.no_grad():
        grad = ops._sdf_grad_tc(_lib.load(), full, p, P)[1].clone()
        o4 = ops.tc_mlp_forward(net.deformer.defs[0].fused(H.RATIO), p, ch=4, conds=defconds[0],
                                batch_inds=bi64).view(P, 4, 3)
        M = _lbs_matrices(net, p + o4[:, 0], bi64, defconds)
    return grad, o4, M


def _pinned(grad, o4, M, R0=None):
    """float64 restatement of sr_tc_shade_point_deformed on its own fp32 inputs, with the per-row bound of
    test_entry_point_vs_float64 (every J here is far from singular)."""
    eye = torch.eye(3, device=grad.device)
    Q = (eye.unsqueeze(0) + o4[:, 1:].transpose(1, 2)).double()          # fl32(delta + Joff), as the kernel forms it
    J = M.double() @ Q
    assert torch.linalg.det(J).abs().min().item() > 1e-2
    g = grad.double()
    y = torch.linalg.solve(J.transpose(1, 2), g.unsqueeze(-1)).squeeze(-1)
    sv = torch.linalg.svdvals(J)
    kappa = sv[:, 0] / sv[:, 2]
    amp = g.norm(dim=1) / sv[:, 2] / y.norm(dim=1)
    n = y / y.norm(dim=1, keepdim=True)
    if R0 is not None:
        n = n @ (torch.from_numpy(FLIP).to(n) @ R0.double().T).T
    return n, 32 * EPS32 * (kappa * amp + 1.0), J, kappa


def _relu_margin(net, pts, bi, defconds):
    """Per point, the smallest |pre-activation| over the translator's hidden units, in float64."""
    from model.Deformer import MLPTranslator
    tr = net.deformer.defs[0]
    t64 = MLPTranslator(tr.feature_vector_size, tr.multires).to(pts.device)
    t64.load_state_dict(tr.state_dict())
    t64 = t64.double()
    zs = []
    t64.relu.register_forward_hook(lambda m, i, o: zs.append(i[0].detach().abs().min(1).values))
    with torch.enable_grad():
        t64(pts.double().requires_grad_(), defconds[0].double(), bi, ratio=H.RATIO)
    return torch.stack(zs).min(0).values


def _cells(net, pp):
    """Skinning cell of p' (lbs.cuh make_axis_f, align_corners=False), [P,3] integers."""
    sk = net.deformer.defs[1]
    D, Hh, W = sk.ws.shape[-3:]
    size = torch.tensor([W, Hh, D], dtype=torch.float64, device=pp.device)
    bmin, bmax = sk.b_min.view(1, 3).double(), sk.b_max.view(1, 3).double()
    x = (((pp.double() - bmin) * 2. / (bmax - bmin)) * size - 1.) / 2.
    return torch.floor(x.clamp(min=0.)).long()


def test_scene_deformed_normals_vs_float64_and_ffma():
    H.dropin()
    import utils
    from selfreconcode_b200 import ops
    net, data, fids = _net()
    pts, rays, bi, defconds, cams = _traced(net, fids)
    P = pts.shape[0]
    assert P >= ops.TC_MIN_POINTS
    R0 = cams.R[0].detach()
    with torch.no_grad():
        n, cr, rgb, dn = utils.shade_rays(net.sdf, net.deformer, net.netRender, pts, rays, defconds, bi, H.RATIO,
                                          deformed_normals=True)
        n0, cr0, rgb0 = utils.shade_rays(net.sdf, net.deformer, net.netRender, pts, rays, defconds, bi, H.RATIO)
        _, _, _, dnr = utils.shade_rays(net.sdf, net.deformer, net.netRender, pts, rays, defconds, bi, H.RATIO,
                                        deformed_normals=True, cam_R0=R0)
        ref, _ = utils.compute_deformed_normals(net.sdf, net.deformer, pts, defconds, bi, H.RATIO, 'test')
        _, gf, _ = net.sdf.forward_fused(pts, H.RATIO, want_grad=True, want_feat=False)
        net.deformer.forward_fused(pts, defconds, bi, H.RATIO)
        off_f = net.deformer.defs[0].offset.view(-1, 3).clone()
    assert torch.equal(n, n0) and torch.equal(cr, cr0) and torch.equal(rgb, rgb0)   # the opt-in changes nothing else
    # (1) the kernel on its own inputs, float64
    grad, o4, M = _kernel_inputs(net, pts, bi, defconds)
    n64, bound, J64, kappa = _pinned(grad, o4, M)
    n64r, _, _, _ = _pinned(grad, o4, M, R0)
    e64 = (dn.double() - n64).abs().max(1).values
    e64r = (dnr.double() - n64r).abs().max(1).values
    print("scene: %d traced points, kappa(J) <= %.1f; vs float64 on the kernel's inputs: max |dn| %.2e, max |dn|/bound "
          "%.3f (camera frame %.2e)" % (P, kappa.max().item(), e64.max().item(), (e64 / bound).max().item(),
                                        e64r.max().item()))
    assert torch.all(e64 <= bound) and torch.all(e64r <= bound)
    # (2) against the FFMA engine: template normals in their band; deformed normals in theirs where J's decisions agree
    e_t = (n - torch.nn.functional.normalize(gf, dim=1)).abs().max(1).values
    e = (dn - ref).abs().max(1).values
    e_r = (dnr - utils.camera_normals(ref, R0)).abs().max(1).values
    margin = _relu_margin(net, pts, bi, defconds)
    cell = (_cells(net, pts + o4[:, 0]) != _cells(net, pts + off_f)).any(1)
    sens = (margin < RELU_MARGIN) | cell
    out = e >= DEFN_BAND
    print("  template normals vs FFMA: max |dn| %.2e (bar %.0e); deformed normals: max |dn| %.2e (camera frame %.2e) "
          "over %d decision-insensitive points (band %.0e); decision-sensitive %d (ReLU %d, cell %d), max |dn| %.2e; "
          "points outside the band %d, all decision-sensitive: %s"
          % (e_t.max().item(), NORMAL_BAR, e[~sens].max().item(), e_r[~sens].max().item(), (~sens).sum().item(),
             DEFN_BAND, sens.sum().item(), (margin < RELU_MARGIN).sum().item(), cell.sum().item(),
             e[sens].max().item() if sens.any() else 0., out.sum().item(), bool(torch.all(sens[out]))))
    for i in torch.nonzero(out).view(-1).tolist():
        print("    point %d: |dn| %.2e, relu margin %.2e, cell changes %s, template |dn| %.2e, kappa %.2f"
              % (i, e[i].item(), margin[i].item(), bool(cell[i]), e_t[i].item(), kappa[i].item()))
    assert e_t.max().item() < NORMAL_BAR
    assert e[~sens].max().item() < DEFN_BAND and e_r[~sens].max().item() < DEFN_BAND
    assert sens.double().mean().item() < 0.1 and bool(torch.all(sens[out]))
    # below TC_MIN_POINTS shade_rays takes compute_deformed_normals itself
    m = ops.TC_MIN_POINTS - 1
    with torch.no_grad():
        _, _, _, ds = utils.shade_rays(net.sdf, net.deformer, net.netRender, pts[:m], rays[:m], defconds, bi[:m],
                                       H.RATIO, deformed_normals=True, cam_R0=R0)
        rs, _ = utils.compute_deformed_normals(net.sdf, net.deformer, pts[:m], defconds, bi[:m], H.RATIO, 'test')
    assert torch.equal(ds, utils.camera_normals(rs, R0))


def _mask_modules(monkeypatch):
    for mod in ("pytorch3d", "trimesh", "openmesh"):
        monkeypatch.setitem(sys.modules, mod, None)        # any import of them raises


def _read_ply(path):
    from test_debug_snapshot_cpu import _read_ply as rp
    return rp(path)


def test_forward_writes_the_reference_snapshot(monkeypatch, tmp_path):
    H.dropin()
    _mask_modules(monkeypatch)
    net, data, fids = _net()
    N, Hh, Ww = fids.numel(), data.H, data.W
    V0, F0 = net.discretizeSDF(H.RATIO, None, 0.0)
    V0 = V0.detach().clone()
    rec = {}
    deform, seed, pcl = net._deform, net._mesh_seed, net._pc_silhouette_loss

    def _deform(*a):
        out = deform(*a)
        rec['def'] = out.detach().clone()
        rec['off'] = net.deformer.defs[0].offset.detach().clone().view(N, -1, 3)
        return out

    def _seed(*a):
        rec['seed'] = seed(*a)
        return rec['seed']

    def _pcl(*a):
        r = pcl(*a)
        rec['masks'], rec['mgt'] = r[1].detach().clone(), r[2].clone()
        return r
    monkeypatch.setattr(net, "_deform", _deform)
    monkeypatch.setattr(net, "_mesh_seed", _seed)
    monkeypatch.setattr(net, "_pc_silhouette_loss", _pcl)
    datas = _datas(N, Hh, Ww)
    quiet, plain, drawn = (os.path.join(tmp_path, d) for d in ("none", "plain", "drawn"))
    torch.manual_seed(5)
    net.forward(datas, 2048, H.RATIO, fids, root=plain)       # remesh step
    names = {'tmp.ply'} | {'%s_%d.ply' % (k, i) for k in ('def', 'def1') for i in range(N)} | \
        {'%s%d.png' % (k, i) for k in ('m', 'mgm') for i in range(N)}
    assert set(os.listdir(plain)) == names
    net.forward(datas, 2048, H.RATIO, fids, root=quiet)       # not a remesh step: nothing
    assert net.forward_time % net.remesh_intersect != 0 and not os.path.exists(quiet)
    # a remesh step with draw, then one with root None
    net.forward_time = 0
    net.draw = True
    torch.manual_seed(5)
    net.forward(datas, 2048, H.RATIO, fids, root=drawn)
    assert net.draw is False
    assert set(os.listdir(drawn)) == names | {'%s%d.png' % (k, i) for k in ('rgb', 'gtrgb', 'normal') for i in range(N)}
    # files of the drawn step against what the step computed
    v, f = _read_ply(os.path.join(drawn, 'tmp.ply'))
    assert v.tobytes() == V0.cpu().numpy().tobytes() and np.array_equal(f, F0.cpu().numpy())
    for i in range(N):
        v, f = _read_ply(os.path.join(drawn, 'def_%d.ply' % i))
        assert v.tobytes() == rec['def'][i].cpu().numpy().tobytes() and np.array_equal(f, F0.cpu().numpy())
        v, _ = _read_ply(os.path.join(drawn, 'def1_%d.ply' % i))
        assert v.tobytes() == (V0 + rec['off'][i]).cpu().numpy().tobytes()
        m = cv2.imread(os.path.join(drawn, 'm%d.png' % i), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(m, (rec['masks'][i] * 255.).cpu().numpy().astype(np.uint8)[..., 0])
        m = cv2.imread(os.path.join(drawn, 'mgm%d.png' % i), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(m, (rec['mgt'][i] * 255.).cpu().numpy().astype(np.uint8))
    # rgb: infer_rays' colours for the same seed; normal: the float64 restatement of the kernel on its own inputs at
    # the draw's traced points, composed the same way; within its bound (~1e-6) the truncating cast moves at most 1 level
    from model import snapshot as S
    bi, ri, ci, ps, _ = rec['seed']
    direct = net.infer_rays(bi, ri, ci, ps, Hh, Ww, H.RATIO, fids).cpu().numpy().astype(np.uint8)
    pts, rays, bi2, defconds, cams = _traced_from_seed(net, fids, bi, ri, ci, ps)
    grad, o4, M = _kernel_inputs(net, pts, bi2, defconds)
    n64, bound, _, _ = _pinned(grad, o4, M, cams.R[0].detach())
    tn = (n64 * 0.5 + 0.5) * 255.
    want = torch.full((N, Hh, Ww, 3), 255., dtype=torch.float64, device=DEV)
    want[bi, ri, ci, :] = tn[:, [2, 1, 0]]
    want_n = want.cpu().numpy().astype(np.uint8)
    lv = 0
    for i in range(N):
        rgb = cv2.imread(os.path.join(drawn, 'rgb%d.png' % i), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(rgb, direct[i])
        gt = cv2.imread(os.path.join(drawn, 'gtrgb%d.png' % i), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(gt, S.gt_color_image(datas['img'][i]))
        nim = cv2.imread(os.path.join(drawn, 'normal%d.png' % i), cv2.IMREAD_UNCHANGED)
        lv = max(lv, int(np.abs(nim.astype(np.int32) - want_n[i]).max()))
    covered = np.zeros((N, Hh, Ww), bool)
    covered[bi.cpu().numpy(), ri.cpu().numpy(), ci.cpu().numpy()] = True
    print("snapshot: %d seed pixels; normal images within %d level of the float64 restatement (bound %.1e)"
          % (covered.sum(), lv, bound.max().item()))
    assert covered.sum() > 500 and lv <= 1 and bound.max().item() < 1e-4
    # root None writes nothing anywhere
    net.forward_time = 0
    net.draw = True
    before = set(os.listdir(tmp_path))
    net.forward(datas, 2048, H.RATIO, fids)
    assert set(os.listdir(tmp_path)) == before and net.draw is True


def _traced_from_seed(net, fids, bi, ri, ci, ps):
    import utils
    N = fids.numel()
    cams, _, _ = net._cameras(N, DEV)
    poses, trans, d_cond, _ = net.dataset.get_grad_parameters(fids, DEV)
    defconds = [d_cond.detach(), [poses.detach(), trans.detach()]]
    with torch.no_grad():
        pix = torch.cat([ci.view(-1, 1), ri.view(-1, 1), torch.ones_like(ci.view(-1, 1))], dim=-1)
        rays = cams.view_rays(pix.float())
    # with autograd on: a user-supplied SDF traces by autograd w.r.t. the points
    pts, _ = utils.OptimizeSurfacePs(cams.cam_pos().detach(), rays, ps.clone(), bi, net.sdf, H.RATIO, net.deformer,
                                     defconds, dthreshold=1.e-4, athreshold=net.angThred, w1=3.05, w2=1., times=30)
    return pts.detach(), rays, bi, defconds, cams


def _run(root, draw, monkeypatch):
    net, data, fids = _net()
    N, Hh, Ww = fids.numel(), data.H, data.W
    net.draw = draw
    if root is not None:
        save = net.save_debug

        def _checked(*a):
            grads = [None if p.grad is None else p.grad.clone() for p in list(net.parameters()) + [net.TmpVs]]
            save(*a)
            after = [None if p.grad is None else p.grad for p in list(net.parameters()) + [net.TmpVs]]
            assert all((x is None and y is None) or torch.equal(x, y) for x, y in zip(grads, after)), \
                "the snapshot touched a gradient"
        monkeypatch.setattr(net, "save_debug", _checked)
    datas = _datas(N, Hh, Ww)
    torch.manual_seed(5)
    loss = net.forward(datas, 2048, H.RATIO, fids, root=root)
    info = repr(net.info)
    rng = (torch.get_rng_state().clone(), torch.cuda.get_rng_state().clone())
    loss.backward()
    net.propagateTmpPsGrad(fids, H.RATIO)
    torch.cuda.synchronize()
    grads = {k: p.grad.clone() for k, p in list(net.named_parameters()) + list(data.named_parameters())
             if p.grad is not None}
    return loss.detach().clone(), info, rng, grads, net.TmpVs.detach().clone(), net.TmpVs.grad.clone()


def test_snapshot_does_not_change_the_step(monkeypatch, tmp_path):
    H.dropin()
    _mask_modules(monkeypatch)
    # torch's index_add / index_select backward sum with atomics unless deterministic algorithms are on (the colour
    # loss's per-frame mean, the latent-code and pose gradients); uninitialised memory is left as the step leaves it
    import torch.utils.deterministic as tud
    was, fill = torch.are_deterministic_algorithms_enabled(), tud.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True, warn_only=True)
    tud.fill_uninitialized_memory = False
    try:
        a = _run(os.path.join(tmp_path, "dbg"), True, monkeypatch)
        b = _run(None, False, monkeypatch)
    finally:
        torch.use_deterministic_algorithms(was)
        tud.fill_uninitialized_memory = fill
    assert len(os.listdir(os.path.join(tmp_path, "dbg"))) == 1 + 7 * 3
    assert torch.equal(a[0], b[0]), (a[0].item(), b[0].item())
    assert a[1] == b[1]
    assert torch.equal(a[2][0], b[2][0]) and torch.equal(a[2][1], b[2][1])
    assert a[3].keys() == b[3].keys() and len(a[3]) > 0
    for k in a[3]:
        assert torch.equal(a[3][k], b[3][k]), k
    assert torch.equal(a[4], b[4]) and torch.equal(a[5], b[5])


class _PlainSdf(torch.nn.Module):
    """The synthetic SDF behind the interface a user-supplied field module offers (forward, gradient, rendcond): no
    fused or tensor-core entry points, so the step traces and shades through autograd."""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner
        self.rendcond = None

    def forward(self, x, ratio):
        out = self.inner(x, ratio)
        self.rendcond = self.inner.rendcond
        return out

    def gradient(self, x, y):
        return self.inner.gradient(x, y)


def test_draw_with_user_supplied_sdf(monkeypatch, tmp_path):
    H.dropin()
    _mask_modules(monkeypatch)
    import utils
    from model import snapshot as S
    net, data, fids = _net()
    net.sdf = _PlainSdf(net.sdf)
    N, Hh, Ww = fids.numel(), data.H, data.W
    rec = {}
    seed = net._mesh_seed

    def _seed(*a):
        rec['seed'] = seed(*a)
        return rec['seed']
    monkeypatch.setattr(net, "_mesh_seed", _seed)
    datas = _datas(N, Hh, Ww)
    root = os.path.join(tmp_path, "dbg")
    net.draw = True
    torch.manual_seed(5)
    loss = net.forward(datas, 2048, H.RATIO, fids, root=root)
    assert torch.isfinite(loss) and net.draw is False
    assert {'%s%d.png' % (k, i) for k in ('rgb', 'gtrgb', 'normal') for i in range(N)} <= set(os.listdir(root))
    loss.backward()
    net.propagateTmpPsGrad(fids, H.RATIO)
    bi, ri, ci, ps, _ = rec['seed']
    direct = net.infer_rays(bi, ri, ci, ps, Hh, Ww, H.RATIO, fids).cpu().numpy().astype(np.uint8)
    pts, rays, bi2, defconds, cams = _traced_from_seed(net, fids, bi, ri, ci, ps)
    with torch.enable_grad():
        ref, _ = utils.compute_deformed_normals(net.sdf, net.deformer, pts.requires_grad_(), defconds, bi2, H.RATIO,
                                                'test')
    want_n = S.normal_image(utils.camera_normals(ref.detach(), cams.R[0].detach()), bi, ri, ci, datas['img'])
    lv = 0
    for i in range(N):
        assert np.array_equal(cv2.imread(os.path.join(root, 'rgb%d.png' % i), cv2.IMREAD_UNCHANGED), direct[i])
        nim = cv2.imread(os.path.join(root, 'normal%d.png' % i), cv2.IMREAD_UNCHANGED)
        lv = max(lv, int(np.abs(nim.astype(np.int32) - want_n[i]).max()))
    print("user-supplied SDF: %d seed pixels drawn; normal images within %d level of compute_deformed_normals"
          % (bi.numel(), lv))
    assert lv <= 1
