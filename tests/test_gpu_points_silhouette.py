"""GPU: the device soft point silhouette (csrc/points_silhouette.cu, ops.points_silhouette) against the float64
restatement of pytorch3d's rule (tests/points_silhouette_ref.py), and OptimNetwork.forward with the built-in point
renderer, across a hierarchy switch, with pytorch3d unimportable.

The restatement is fed the device's own fp32 screen coordinates, so both sides take the same decisions except within
rounding of one.  Bars: mask |a-b| <= 1e-5; gradient w.r.t. the deformed template helpers.elem_err < 1e-4 over the
points not within rounding of a decision (|d2 - r^2| <= 1e-6 r^2 at some pixel, or a depth tie at a K-th slot; these
are counted and printed).  Negative controls must fail those bars."""
import ctypes as C
import sys

import numpy as np
import pytest
import torch

import helpers as H
import points_silhouette_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _template(Hh, Ww, n_frames):
    """The synthetic template deformed into n_frames frames (leaf tensor) and the frames' cameras."""
    from test_gpu_mesh_shade import _scene
    net, data, cams, TmpVs, Tmpfs, fids = _scene(Hh, Ww, n_frames)
    poses, trans, d_cond, _ = data.get_grad_parameters(fids, DEV)
    with torch.no_grad():
        dv = net.deformer(TmpVs[None].expand(n_frames, -1, 3), [d_cond, [poses, trans]], ratio=H.RATIO)
    return dv.detach().contiguous(), cams


def _cotangent(N, Hh, Ww, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(N, Hh, Ww, generator=g, dtype=torch.float64).numpy()


def _device(x, Hh, Ww, r, K, G, cams=None):
    """mask [N,H,W], dL/dx for L = sum G * mask; x = world vertices (with cams) or screen points."""
    from selfreconcode_b200 import ops
    H.dropin()
    from model.raster import screen_vertices
    x = x.detach().clone().requires_grad_(True)
    pts = screen_vertices(x, cams) if cams is not None else x
    m = ops.points_silhouette(pts, Hh, Ww, r, K)
    g, = torch.autograd.grad((m[..., 0] * torch.from_numpy(G).float().to(DEV)).sum(), [x])
    torch.cuda.synchronize()
    return m[..., 0].detach(), g, pts.detach()


def _ref_grad(x, g_screen, cams):
    """Chain a screen-space cotangent [N,V,3] to x through the same projection (identity for screen points)."""
    H.dropin()
    from model.raster import screen_vertices
    gs = torch.from_numpy(g_screen).float().to(DEV)
    if cams is None:
        return gs
    x = x.detach().clone().requires_grad_(True)
    return torch.autograd.grad(screen_vertices(x, cams), [x], gs)[0]


def _check(name, x, Hh, Ww, r, K, cams=None, seed=0):
    G = _cotangent(x.shape[0], Hh, Ww, seed)
    m, g, pts = _device(x, Hh, Ww, r, K, G, cams)
    m2, g2, _ = _device(x, Hh, Ww, r, K, G, cams)
    assert torch.equal(m, m2) and torch.equal(g, g2), "reruns must be bit-identical"
    r32 = float(np.float32(r))
    ndc = ref.screen_to_ndc(pts.cpu().numpy(), Hh, Ww)
    mref = ref.silhouette(ndc, Hh, Ww, r32, K)
    merr = np.abs(m.cpu().numpy() - mref).max()
    gref = _ref_grad(x, ref.ndc_grad_to_screen(ref.silhouette_grad(ndc, Hh, Ww, r32, K, G), Hh, Ww), cams)
    skip = ref.borderline_points(ndc, Hh, Ww, r32, K)
    keep = ~skip.reshape(-1)
    gd, gr = g.cpu().numpy().reshape(-1, 3), gref.cpu().numpy().reshape(-1, 3)
    gerr = H.elem_err(gd[keep], gr[keep])
    P = ref.rasterize(ndc, Hh, Ww, r32, None)
    print("%s: %d frames x %d points, %dx%d, r=%g, K=%d: %d covered pixels, max %d points on a pixel; mask max |err| "
          "%.2e; gradient elem_err %.2e over %d points (%d within rounding of a decision excluded)"
          % (name, x.shape[0], x.shape[1], Hh, Ww, r, K, int((mref > 0).sum()), int(P["n_cover"].max()), merr, gerr,
             int(keep.sum()), int(skip.sum())))
    assert merr <= 1e-5 and gerr < 1e-4
    assert (mref > 0).sum() > 100 and np.abs(gr[keep]).max() > 0
    return dict(m=m.cpu().numpy(), ndc=ndc, G=G, gd=gd, keep=keep, r32=r32, x=x, cams=cams)


def test_template_square_three_frames():
    dv, cams = _template(512, 512, 3)
    _check("template 512x512", dv, 512, 512, 0.006, 50, cams)


def test_template_non_square():
    dv, cams = _template(112, 96, 3)
    c = _check("template 112x96", dv, 112, 96, 0.03, 50, cams, seed=1)
    # negative control: isotropic pixels (NDC scaled by the shorter side) is a different rule on this image
    iso = np.abs(c["m"] - ref.silhouette(c["ndc"], 112, 96, c["r32"], 50, isotropic=True)).max()
    print("   isotropic-pixel control: mask max |err| %.2e" % iso)
    assert iso > 1e-5


def crowded_scene():
    """Two frames of screen points on a 32x32 image at r = 0.15 (2.4 pixels): a stack of 60 coincident points with
    depths repeating in threes (more than K = 50 on every pixel it covers, ties at the K-th slot), two points exactly
    on the centre of pixel (20, 20) and one on (20, 21) (w = 1 factors), points behind the camera, and scattered
    points on a 1/16-pixel lattice (no coverage decision within rounding)."""
    g = np.random.default_rng(7)
    pts = [[10.25, 12.5, 1.0 + 0.01 * (k % 20)] for k in range(60)]
    pts += [[20.0, 20.0, 1.5], [20.0, 20.0, 2.0], [21.0, 20.0, 1.0], [20.5, 20.25, 1.2]]
    pts += [[12.0, 12.0, -0.5], [20.0, 20.0, -1.0]]
    scat = np.stack([np.round(g.uniform(0, 31, 80) * 16) / 16, np.round(g.uniform(0, 31, 80) * 16) / 16,
                     g.uniform(0.5, 3.0, 80)], 1)
    f0 = np.concatenate([np.array(pts), scat])
    f1 = f0 + np.array([3.5, -2.25, 0.0])
    return torch.from_numpy(np.stack([f0, f1])).float().to(DEV).contiguous()


def test_crowded_scene_and_controls():
    x = crowded_scene()
    c = _check("crowded 32x32", x, 32, 32, 0.15, 50, seed=2)
    m, ndc, G, r32 = c["m"], c["ndc"], c["G"], c["r32"]
    assert m[0, 20, 20] >= 1.0 - 1e-6 and m[0, 20, 21] >= 1.0 - 1e-6       # w = 1 factors
    # negative controls: every covering point composited (no K truncation); w without the 1/r^2; the gradient
    # without the prod_{q != p} (1 - w_q) factor
    c1 = np.abs(m - ref.silhouette(ndc, 32, 32, r32, None)).max()
    c2 = np.abs(m - ref.silhouette(ndc, 32, 32, r32, 50, r2_scale=False)).max()
    g_no = ref.ndc_grad_to_screen(ref.silhouette_grad(ndc, 32, 32, r32, 50, G, with_others=False), 32, 32)
    c3 = H.elem_err(c["gd"][c["keep"]], g_no.reshape(-1, 3)[c["keep"]])
    print("   controls: no K truncation %.2e, w without 1/r^2 %.2e, gradient without prod_{q!=p} %.2e" % (c1, c2, c3))
    assert c1 > 1e-5 and c2 > 1e-5 and c3 > 1e-4


def test_invalid_arguments():
    from selfreconcode_b200 import _lib, ops
    lib = _lib.load()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.zeros(4096, device=DEV)
    p = C.c_void_p(buf.data_ptr())
    z = C.c_void_p(0)
    cap = lib.sr_points_silhouette_list_capacity
    assert cap(1, 4, 8, 8, 0.1) > 0
    for a in ((0, 4, 8, 8, 0.1), (1, 0, 8, 8, 0.1), (1, 4, 0, 8, 0.1), (1, 4, 8, -1, 0.1), (1, 4, 8, 8, 0.0),
              (1, 4, 8, 8, -0.1), (1, 4, 8, 8, float("inf")), (1, 4, 8, 8, float("nan"))):
        assert cap(*a) == _lib.SR_EINVAL, a
    good = dict(bin=[p, p, 1, 4, 8, 8, 0.1, p, p, s],
                forward=[p, p, p, 1, 4, 8, 8, 0.1, 3, p, p, p, p, s],
                backward=[p, p, p, p, p, 1, 4, 8, 8, 0.1, p, s])
    ptrs = dict(bin=(0, 1, 7, 8), forward=(0, 1, 2, 9, 10, 11, 12), backward=(0, 1, 2, 3, 4, 10))
    sizes = dict(bin=(2, 3, 4, 5), forward=(3, 4, 5, 6), backward=(5, 6, 7, 8))
    rad = dict(bin=6, forward=7, backward=9)
    for k, fn in (("bin", lib.sr_points_silhouette_bin), ("forward", lib.sr_points_silhouette_forward),
                  ("backward", lib.sr_points_silhouette_backward)):
        for i in ptrs[k]:
            a = list(good[k])
            a[i] = z
            assert fn(*a) == _lib.SR_EINVAL, (k, i)
        for i in sizes[k]:
            for bad in (0, -1):
                a = list(good[k])
                a[i] = bad
                assert fn(*a) == _lib.SR_EINVAL, (k, i, bad)
        for bad in (0.0, -1.0, float("inf"), float("nan")):
            a = list(good[k])
            a[rad[k]] = bad
            assert fn(*a) == _lib.SR_EINVAL, (k, bad)
    for bad in (0, -2):
        a = list(good["forward"])
        a[8] = bad
        assert lib.sr_points_silhouette_forward(*a) == _lib.SR_EINVAL
    with pytest.raises(ValueError):
        ops.points_silhouette(torch.zeros(1, 4, 3, device=DEV), 8, 8, 0.0, 5)
    with pytest.raises(ValueError):
        ops.points_silhouette(torch.zeros(1, 4, 3, device=DEV), 8, 8, 0.1, 0)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# OptimNetwork.forward end to end
# ---------------------------------------------------------------------------------------------------------------------
class _RefSilhouette(torch.autograd.Function):
    """The restatement as an autograd function of the screen points (float64 on the host)."""

    @staticmethod
    def forward(ctx, pts, Hh, Ww, r, K):
        ndc = ref.screen_to_ndc(pts.detach().cpu().numpy(), Hh, Ww)
        ctx.args = (ndc, Hh, Ww, r, K)
        return torch.from_numpy(ref.silhouette(ndc, Hh, Ww, r, K)).float().to(pts.device)[..., None]

    @staticmethod
    def backward(ctx, g):
        ndc, Hh, Ww, r, K = ctx.args
        gn = ref.silhouette_grad(ndc, Hh, Ww, r, K, g[..., 0].double().cpu().numpy())
        return torch.from_numpy(ref.ndc_grad_to_screen(gn, Hh, Ww)).float().to(g.device), None, None, None, None


class _RefRenderer:
    takes_tensors = True

    def __init__(self, builtin):
        self.rasterizer = builtin.rasterizer
        self.radius = builtin.radius

    def __call__(self, verts):
        from model.raster import screen_vertices
        s = self.rasterizer.raster_settings
        pts = screen_vertices(verts, self.rasterizer.cameras)
        return _RefSilhouette.apply(pts, s.image_size[0], s.image_size[1], float(np.float32(s.radius)),
                                    s.points_per_pixel)


def _step(use_ref, Hh, Ww):
    import utils
    from selfreconcode_b200 import synth
    from test_gpu_mesh_shade import _gts, _scene
    from model.raster import PointsSilhouetteRenderer
    net, data, cams, _, _, fids = _scene(Hh, Ww, 3)
    conf = synth.reference_config()
    conf._find('train.coarse.point_render')['radius'] = 0.02     # 1.3 pixels at 128x128
    for lvl in ('loss_coarse', 'loss_medium', 'loss_fine'):
        # mesh regulariser weights <= 0, as config.conf ships them
        conf[lvl] = dict(conf[lvl], pc_weight=dict(weight=60., mask_weight=1., laplacian_weight=-10.,
                                                   edge_weight=-10., norm_weight=-0.001,
                                                   def_consistent=dict(weight=0.1, c=0.005)))
    loader = torch.utils.data.DataLoader(list(range(3)), 3)
    net, loader = utils.set_hierarchical_config(conf, 'coarse', net, loader, synth.MC_LADDER_65)
    net.update_hierarchical_config(torch.device(DEV))
    assert isinstance(net.pcRender, PointsSilhouetteRenderer) and net.pcRender.radius == 0.02
    if use_ref:
        net.pcRender = _RefRenderer(net.pcRender)
    V0 = net.discretizeSDF(H.RATIO, None, 0.0)[0].detach().clone()
    g = torch.Generator().manual_seed(21)
    datas = {'img': (torch.rand(3, Hh, Ww, 3, generator=g) * 2 - 1).to(DEV),
             'mask': _gts(3, Hh, Ww, image=False)['mask']}
    torch.manual_seed(5)
    loss = net.forward(datas, 2048, H.RATIO, fids)
    info = dict(net.info)
    # the inner step is SGD's first (momentum buffer = gradient): displacement = -lr * grad, taken from the gradient
    # because TmpVs - V0 loses ~6e-8 absolute to fp32 cancellation against displacements of ~1e-5
    disp = (-0.05 * net.TmpVs.grad.detach()).cpu().numpy()
    assert net.TmpVs.shape == V0.shape
    assert np.abs((net.TmpVs.detach() - V0).cpu().numpy() - disp).max() <= 2e-7
    loss.backward()
    net.propagateTmpPsGrad(fids, H.RATIO)
    torch.cuda.synchronize()
    return info, disp, loss.item()


def test_forward_step_without_pytorch3d(monkeypatch):
    H.dropin()
    monkeypatch.setitem(sys.modules, "pytorch3d", None)        # any pytorch3d import raises
    with pytest.raises(ImportError):
        import pytorch3d  # noqa: F401
    Hh = Ww = 128
    info, disp, loss = _step(False, Hh, Ww)
    info_r, disp_r, loss_r = _step(True, Hh, Ww)
    ml, ml_r = info['pc_loss']['mask_loss'], info_r['pc_loss']['mask_loss']
    derr = H.elem_err(disp, disp_r)
    print("forward step: mask_loss %.7f (restatement %.7f, |diff| %.2e); TmpVs displacement elem_err %.2e "
          "(max |displacement| %.2e over %d vertices); loss %.6f / %.6f"
          % (ml, ml_r, abs(ml - ml_r), derr, np.abs(disp_r).max(), disp.shape[0], loss, loss_r))
    assert 0.0 < ml < 1.0 and 'skipped' not in info['pc_loss']
    assert abs(ml - ml_r) <= 1e-5
    assert np.abs(disp_r).max() > 0 and derr < 1e-4
