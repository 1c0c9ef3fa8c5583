"""GPU: the textured avatar (csrc/avatar_texture.cu, selfreconcode_b200.avatar) against the float64 restatement
(tests/avatar_texture_ref.py) and exact invariants: kernels vs restatement, the affine invariant, coverage weighting,
a round trip through the baker, reposing, the export's skinning, and the written outputs.  Scenes: the synthetic
template of test_gpu_mesh_shade._scene with the UV layouts of test_gpu_texture.

Bars (measured on one H100 beside them): mips per level <= 1e-6 (1.4e-7), shaded output <= 2e-5 (1.6e-7), affine
invariant <= 0.6/255 (0.28/255), chart colour under coverage weighting <= 1/255 (0), round trip p99 <= 8/255 (6/255),
pose_vertices + yaw 360 <= 1e-5 (0), distances to the turn axis <= 1e-5 (1.2e-7), random poses vs float64 translator +
LBS <= 2e-5 (8.9e-7), export LBS <= 1e-5 (3.6e-7), skin-weight row sums <= 1e-5 (3.1e-7)."""
import os
import types

import numpy as np
import pytest
import torch

import avatar_texture_ref as ref
import grid_sampler_ref
import helpers as H
from test_gpu_texture import chart_layout, g_colour, scene, seam_layout, write_obj

pytestmark = pytest.mark.gpu
DEV = "cuda"

_SCENES = {}


def scene_hw(Hh, Ww, n):
    """(net, data, cams, TmpVs, Tmpfs) of a non-square image, root rotations as test_gpu_texture.scene."""
    if (Hh, Ww, n) not in _SCENES:
        from test_gpu_mesh_shade import _scene
        net, data, cams, TmpVs, Tmpfs, _ = _scene(Hh, Ww, n)
        with torch.no_grad():
            data.poses[:, 0, 1] = torch.linspace(-0.6, 0.6, n, device=DEV)
        _SCENES[(Hh, Ww, n)] = (net, data, cams, TmpVs, Tmpfs.long())
    return _SCENES[(Hh, Ww, n)]


def fragments(net, data, cams, TmpVs, Tmpfs, n):
    from selfreconcode_b200 import ops
    from selfreconcode_b200.avatar import pose_vertices
    H.dropin()
    from model.raster import screen_vertices
    ids = torch.arange(n, device=DEV)
    poses, trans, d_cond, _ = data.get_grad_parameters(ids, DEV)
    D = pose_vertices(net, TmpVs, poses, trans, d_cond)
    s = screen_vertices(D, cams).contiguous()
    p2f, bary, _ = ops.raster_mesh(s, Tmpfs, data.H, data.W)
    return s, p2f[..., 0], bary[..., 0, :]


def mixed_texture(R, seed=0):
    """Smooth gradients plus a high-frequency checker and noise, [R,R,3] uint8."""
    yy, xx = np.meshgrid(np.arange(R, dtype=np.float64), np.arange(R, dtype=np.float64), indexing="ij")
    smooth = 127.5 + 90. * np.stack([np.sin(xx / 23. + c) * np.cos(yy / 31. - c) for c in range(3)], -1)
    checker = 60. * (((xx // 2 + yy // 2) % 2) * 2 - 1)[..., None]
    noise = np.random.default_rng(seed).normal(0, 25., (R, R, 3))
    hf = (xx > R / 2)[..., None]
    return np.clip(np.rint(smooth + np.where(hf, checker + noise, 0.)), 0, 255).astype(np.uint8)


def device_levels(mips, levels):
    out = []
    for off, h, w in levels.tolist():
        out.append(mips[off:off + h * w].view(h, w, 4).double().cpu().numpy())
    return out


# ---- 1. kernels vs restatement ------------------------------------------------------------------------------------
@pytest.mark.parametrize("Hh,Ww", [(36, 40), (120, 96), (960, 832)])
def test_kernels_vs_restatement(Hh, Ww):
    from selfreconcode_b200 import ops
    from selfreconcode_b200.texture import uv_raster
    net, data, cams, TmpVs, Tmpfs = scene_hw(Hh, Ww, 3)
    R = 420
    vt, ft = chart_layout(Tmpfs.shape[0])
    vt_d, ft_d = torch.from_numpy(vt).to(DEV), torch.from_numpy(ft).to(DEV)
    tex = mixed_texture(R)
    cov = uv_raster(vt_d, ft_d, R, R)[0] >= 0
    tex_d = torch.from_numpy(tex).to(DEV)
    mips, levels = ops.texture_mips(tex_d, cov)
    mips2, _ = ops.texture_mips(tex_d, cov)
    lv_ref = ref.mips(tex, cov.cpu().numpy())
    lv_dev = device_levels(mips, levels)
    assert len(lv_ref) == len(lv_dev) == levels.shape[0]
    m_err = max(float(np.abs(a - b).max()) for a, b in zip(lv_dev, lv_ref))
    s, p2f, bary = fragments(net, data, cams, TmpVs, Tmpfs, 3)
    bg_img = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (3, Hh, Ww, 3), dtype=np.uint8)).to(DEV)
    errs, lams = [], None
    for bg in ((0.25, 0.5, 1.0), bg_img):
        out = ops.shade_textured(p2f, bary, s, Tmpfs, ft_d, vt_d, mips, levels, bg)
        again = ops.shade_textured(p2f, bary, s, Tmpfs, ft_d, vt_d, mips2, levels, bg)
        torch.cuda.synchronize()
        assert torch.equal(out, again) and torch.equal(mips, mips2), "reruns must be bit-identical"
        want, lams = ref.shade(p2f.cpu().numpy(), bary.cpu().numpy(), s.cpu().numpy(), Tmpfs.cpu().numpy(), ft, vt,
                               lv_dev, bg if isinstance(bg, tuple) else bg.cpu().numpy())
        got = out.double().cpu().numpy()
        errs.append(float(np.abs(got - want).max()))
    covered = (p2f >= 0).sum().item()
    print("kernels %dx%d, atlas %d^2, %d levels: mips max |err| %.2e; %d covered pixels, lambda min %.2f median %.2f "
          "max %.2f; shaded max |err| %.2e (colour), %.2e (image background)"
          % (Hh, Ww, R, levels.shape[0], m_err, covered, lams.min(), np.median(lams), lams.max(), *errs))
    assert m_err <= 1e-6
    assert covered > 200
    assert max(errs) <= 2e-5
    if Hh == 36:
        assert np.median(lams) >= 2.             # minified
    if Hh == 960:
        assert (lams == 0.).mean() > 0.05        # magnified: plain bilinear on level 0


# ---- 2. affine invariant ------------------------------------------------------------------------------------------
AFF = np.array([[0.15, 0.6, 0.1], [0.4, -0.3, 0.5], [0.5, 0.2, -0.35]])    # rows: channel = a + b u + c v


def test_affine_invariant():
    from selfreconcode_b200 import ops
    net, data, cams, TmpVs, Tmpfs = scene_hw(160, 144, 2)
    R = 1024
    vt, ft = chart_layout(Tmpfs.shape[0])
    c = (np.arange(R) + 0.5) / R
    u, v = np.meshgrid(c, 1. - c)
    tex = np.clip(np.rint(255. * (AFF[:, 0] + AFF[:, 1] * u[..., None] + AFF[:, 2] * v[..., None])), 0, 255)
    mips, levels = ops.texture_mips(torch.from_numpy(tex.astype(np.uint8)).to(DEV),
                                    torch.ones(R, R, dtype=torch.bool, device=DEV))
    s, p2f, bary = fragments(net, data, cams, TmpVs, Tmpfs, 2)
    vt_d, ft_d = torch.from_numpy(vt).to(DEV), torch.from_numpy(ft).to(DEV)
    out = ops.shade_textured(p2f, bary, s, Tmpfs, ft_d, vt_d, mips, levels).cpu().numpy()
    p = p2f.cpu().numpy()
    cov = p >= 0
    F = Tmpfs.shape[0]
    b = bary.cpu().numpy().astype(np.float64)[cov]
    uvc = vt.astype(np.float64)[ft[p[cov] % F]]
    uu, vv = (b * uvc[..., 0]).sum(-1), (b * uvc[..., 1]).sum(-1)
    want = AFF[:, 0] + AFF[:, 1] * uu[:, None] + AFF[:, 2] * vv[:, None]
    _, lam = ref.shade(p, bary.cpu().numpy(), s.cpu().numpy(), Tmpfs.cpu().numpy(), ft, vt,
                       device_levels(mips, levels), (1., 1., 1.))
    # clamp-to-edge is not affine: keep samples at least half a texel of the coarser level inside the atlas
    L = levels.shape[0]
    Wl = np.array([int(levels[min(int(l) + 1, L - 1), 2]) for l in np.floor(lam)], np.float64)
    inside = (np.minimum(uu, 1 - uu) * Wl >= 0.5) & (np.minimum(vv, 1 - vv) * Wl >= 0.5)
    err = np.abs(out[cov][:, :3] - want).max(1)
    print("affine: %d covered pixels, %d away from the atlas edge at their level; lambda max %.2f; max |err| %.3f/255"
          % (cov.sum(), inside.sum(), lam.max(), 255 * err[inside].max()))
    assert inside.sum() > 0.8 * cov.sum()
    assert err[inside].max() <= 0.6 / 255.


# ---- 3. coverage weighting ----------------------------------------------------------------------------------------
def test_coverage_weighting():
    from selfreconcode_b200 import ops
    from selfreconcode_b200.texture import uv_raster
    net, data, cams, TmpVs, Tmpfs = scene_hw(96, 96, 2)
    vt, ft = chart_layout(Tmpfs.shape[0])
    vt_d, ft_d = torch.from_numpy(vt).to(DEV), torch.from_numpy(ft).to(DEV)
    s, p2f, bary = fragments(net, data, cams, TmpVs, Tmpfs, 2)
    p, bn, sn, fc = p2f.cpu().numpy(), bary.cpu().numpy(), s.cpu().numpy(), Tmpfs.cpu().numpy()
    # the atlas size that puts the median footprint near 16 texels per pixel
    cov = p >= 0
    F = Tmpfs.shape[0]
    corners = sn[(p[cov] // F)[:, None], fc[p[cov] % F]].astype(np.float64)
    n_i, r_i, c_i = np.nonzero(cov)
    rho = ref.footprint(corners[..., :2], 1. / corners[..., 2], vt.astype(np.float64)[ft[p[cov] % F]],
                        c_i.astype(np.float64), r_i.astype(np.float64), 512, 512)
    R = int(np.clip(round(512 * 16. / np.median(rho) / 8) * 8, 64, 4096))
    colour = np.array([40, 180, 220], np.uint8)
    mask = (uv_raster(vt_d, ft_d, R, R)[0] >= 0).cpu().numpy()
    tex = np.where(mask[..., None], colour, 0).astype(np.uint8)
    mips, levels = ops.texture_mips(torch.from_numpy(tex).to(DEV), torch.from_numpy(mask).to(DEV))
    out = ops.shade_textured(p2f, bary, s, Tmpfs, ft_d, vt_d, mips, levels).cpu().numpy()[cov][:, :3]
    lv = device_levels(mips, levels)
    # interior: every tap of both levels has coverage
    _, lam = ref.shade(p, bn, sn, fc, ft, vt, lv, (1., 1., 1.))
    b = bn.astype(np.float64)[cov]
    uvc = vt.astype(np.float64)[ft[p[cov] % F]]
    uu, vv = (b * uvc[..., 0]).sum(-1), (b * uvc[..., 1]).sum(-1)
    L = len(lv)
    interior = np.ones(uu.shape, bool)
    for k in (0, 1):
        l = np.minimum(np.floor(lam).astype(np.int64) + k, L - 1)
        for li in np.unique(l):
            sel = l == li
            w = ref.bilinear(lv[li][..., 3:], uu[sel] * lv[li].shape[1] - 0.5, (1 - vv[sel]) * lv[li].shape[0] - 0.5)
            Hl, Wl = lv[li].shape[:2]
            x, y = uu[sel] * Wl - 0.5, (1 - vv[sel]) * Hl - 0.5
            taps = [lv[li][np.clip(np.floor(y) + dy, 0, Hl - 1).astype(int), np.clip(np.floor(x) + dx, 0, Wl - 1).astype(int), 3]
                    for dy in (0, 1) for dx in (0, 1)]
            interior[sel] &= np.all(np.stack(taps) > 0, 0) & (w[..., 0] > 0)
    err = np.abs(out - colour / 255.).max(1)
    naive = ref.shade(p, bn, sn, fc, ft, vt, ref.mips(tex, np.ones_like(mask)), (1., 1., 1.))[0][cov][:, :3]
    dark = (colour / 255. - naive).max(1)
    print("coverage weighting: atlas %d^2, lambda median %.2f, %d / %d interior pixels; max |err| %.3f/255; "
          "all-ones coverage darkens them by median %.1f/255, min %.1f/255"
          % (R, np.median(lam), interior.sum(), cov.sum(), 255 * err[interior].max(), 255 * np.median(dark[interior]),
             255 * dark[interior].min()))
    assert 2.5 <= np.median(lam) <= 5.5
    assert interior.sum() > 0.5 * cov.sum()
    assert err[interior].max() <= 1. / 255.
    assert np.median(dark[interior]) > 20. / 255.


# ---- 4-7. the avatar on a trained network ---------------------------------------------------------------------------
_SEQ = {}


def sequence(tmp_root, n_frames=8, side=384, R=256):
    """Frames coloured by g (test_gpu_texture.test_round_trip) at the canonical point seen there, written as a sequence;
    the texture baked from them with bake_from_network on the seam layout.  -> dict."""
    key = (n_frames, side, R)
    if key in _SEQ:
        return _SEQ[key]
    from selfreconcode_b200 import ops
    from selfreconcode_b200.texture import bake_from_network, load_obj_uv
    H.dropin()
    from dataset import write_sequence
    from dataset.dataset import SceneDataset
    from model.raster import screen_vertices
    net, data, cams, TmpVs, Tmpfs = scene(side, n_frames)
    vt, ft = seam_layout(TmpVs.cpu().numpy(), Tmpfs.cpu().numpy())
    root = os.path.join(tmp_root, "seq")
    os.makedirs(root, exist_ok=True)
    obj = os.path.join(root, "uvmap.obj")
    write_obj(obj, TmpVs.cpu().numpy(), Tmpfs.cpu().numpy(), vt, ft)
    Vr = load_obj_uv(obj)[0].to(DEV)
    poses, trans, d_cond, _ = data.get_grad_parameters(torch.arange(n_frames, device=DEV), DEV)
    with torch.no_grad():
        D = net.deformer(Vr[None].expand(n_frames, -1, 3), [d_cond, [poses, trans]], ratio={'sdfRatio': 1.,
                         'deformerRatio': 1., 'renderRatio': 1.})
    cn = Vr.double().cpu().numpy()
    fc = Tmpfs.cpu().numpy()
    imgs, masks = [], []
    for n in range(n_frames):
        p2f, bary, _ = ops.raster_mesh(screen_vertices(D[n:n + 1], cams), Tmpfs, side, side)
        p2f, bary = p2f[0, ..., 0].cpu().numpy(), bary[0, ..., 0, :].cpu().numpy().astype(np.float64)
        hit = p2f >= 0
        col = np.full((side, side, 3), 0.2)
        col[hit] = g_colour((bary[hit][:, :, None] * cn[fc[p2f[hit]]]).sum(1))
        imgs.append(np.rint(col * 255.) / 255. * 2. - 1.)
        masks.append(hit.astype(np.float32))
    f, pp = data.focals.detach().view(2).cpu().numpy(), data.pps.detach().view(2).cpu().numpy()
    write_sequence(root, np.stack(imgs), np.stack(masks), data.poses.detach().cpu().numpy(),
                   data.trans.detach().cpu().numpy(), np.zeros(10, np.float32),
                   dict(fx=f[0], fy=f[1], cx=pp[0], cy=pp[1], quat=[0., 0., 0., 1.], T=[0., 0., 0.]))
    ds = SceneDataset(root, {'deformer': 128})
    with torch.no_grad():
        ds.conds[0].copy_(data.conds[0].detach().cpu())
    tnet = types.SimpleNamespace(deformer=net.deformer, dataset=ds)
    tex_dir = os.path.join(root, "template")
    baked = bake_from_network(tnet, obj, tex_dir, num=n_frames, resolution=R, min_views=2)
    _SEQ[key] = dict(net=tnet, data=data, obj=obj, tex=os.path.join(tex_dir, "texture.png"), baked=baked, vt=vt,
                     ft=ft, Vr=Vr, faces=Tmpfs, n=n_frames, side=side, R=R, root=root)
    return _SEQ[key]


@pytest.fixture(scope="module")
def seq(tmp_path_factory):
    return sequence(str(tmp_path_factory.mktemp("avatar")))


def test_round_trip_with_the_baker(seq, tmp_path):
    import cv2
    from selfreconcode_b200 import ops
    from selfreconcode_b200.avatar import TexturedAvatar, pose_vertices, render_sequence
    H.dropin()
    from model.raster import screen_vertices
    net, ds, n, side, R = seq["net"], seq["net"].dataset, seq["n"], seq["side"], seq["R"]
    av = TexturedAvatar(seq["obj"], seq["tex"], DEV)
    assert torch.equal(av.coverage, seq["baked"]["tex_mask"])
    out_dir = str(tmp_path / "render")
    fids, mad, psnr = render_sequence(net, av, out_dir, batch=3)
    assert np.array_equal(fids, np.arange(n))
    poses, trans, d_cond = ds.get_grad_parameters(torch.arange(n), DEV)[:3]
    D = pose_vertices(net, av.V, poses, trans, d_cond)
    f, pp, Rc, Tc, _, _ = ds.get_camera_parameters(n, DEV)
    from model.CameraMine import RectifiedPerspectiveCameras
    cams = RectifiedPerspectiveCameras(f, pp, Rc, Tc)
    s = screen_vertices(D, cams).contiguous()
    p2f, bary, _ = ops.raster_mesh(s, av.faces, side, side)
    p = p2f[..., 0].cpu().numpy()
    cov = p >= 0
    F = av.faces.shape[0]
    b = bary[..., 0, :].cpu().numpy().astype(np.float64)[cov]
    vt, ft = seq["vt"], seq["ft"]
    uvc = vt.astype(np.float64)[ft[p[cov] % F]]
    uu, vv = (b * uvc[..., 0]).sum(-1), (b * uvc[..., 1]).sum(-1)
    mf = seq["baked"]["mask_final"].cpu().numpy()
    ti = np.clip(np.floor((1 - vv) * R), 0, R - 1).astype(int)
    tj = np.clip(np.floor(uu * R), 0, R - 1).astype(int)
    frames = np.stack([cv2.imread(ds.img_ns[i]) for i in range(n)]).astype(np.float64)
    masks = np.stack([cv2.imread(ds.mask_ns[i])[..., 0] > 0 for i in range(n)])
    keep = masks[cov] & mf[ti, tj] & (uu >= 0) & (uu <= 1) & (vv >= 0) & (vv <= 1)
    rendered = np.stack([cv2.imread(os.path.join(out_dir, "%d.png" % i)) for i in range(n)]).astype(np.float64)

    def p99(img):
        return float(np.quantile(np.abs(img[cov][keep] - frames[cov][keep]).max(1), 0.99))

    atlas = cv2.imread(seq["tex"])
    lv = ref.mips(atlas, av.coverage.cpu().numpy())
    args = (p, bary[..., 0, :].cpu().numpy(), s.cpu().numpy(), av.faces.cpu().numpy(), ft, vt, lv, (0., 0., 0.))
    ctl = {k: np.rint(np.clip(ref.shade(*args, **kw)[0][..., :3], 0, 1) * 255.)
           for k, kw in (("v not flipped", dict(flip_v=False)), ("half texel", dict(texel_shift=0.5)))}
    # magnified pixels only (plain bilinear on level 0): where the footprint spans several texels the render is the
    # filtered atlas, while a frame pixel is g at one point
    lam = ref.shade(*args)[1]
    n_min = int(keep.sum())
    keep &= lam == 0.
    e = p99(rendered)
    print("round trip: %d frames %d^2, atlas %d^2, %d pixels with a final texel, %d of them magnified; p99 %.2f/255; "
          "controls: %s; mad mean %.2f, psnr mean %.2f" % (n, side, R, n_min, keep.sum(), e, ", ".join("%s p99 %.2f/255" % (k, p99(v)) for k, v in ctl.items()),
                              mad.mean(), psnr.mean()))
    # Bar from measurement (one H100): p99 6/255 over 103 625 magnified pixels (the controls: 20/255 half a texel off,
    # 203/255 with v not flipped).  It is the bake's own error at 8 views (outline and self-occlusion samples kept in a
    # texel's median, test_gpu_texture.test_round_trip) plus two resamplings and three uint8 roundings; the shader's own
    # error is bounded by test_kernels_vs_restatement.
    assert n_min > 0.5 * cov.sum() and keep.sum() > 5000
    assert e <= 8.
    for k, v in ctl.items():
        assert p99(v) > 8., k


def _turn_axis(ds):
    R = ds.get_camera_parameters(1, DEV)[2].reshape(3, 3).double().cpu().numpy()
    return R[:, 1] / np.linalg.norm(R[:, 1])


def translator_f64(tr, pts, cond):
    """The translator's MLP in float64 at ratio 1 (positional weights 1): pts [P,3], cond [C] -> offsets [P,3]."""
    x = pts.double()
    parts = [x]
    for k in range(tr.multires):
        parts += [torch.sin(x * 2. ** k), torch.cos(x * 2. ** k)]
    h = torch.cat(parts + [cond.double().view(1, -1).expand(x.shape[0], -1)], 1)
    for l in range(tr.num_layers - 1):
        lin = getattr(tr, "lin%d" % l)
        h = h @ lin.weight.double().t() + lin.bias.double()
        if l < tr.num_layers - 2:
            h = torch.relu(h)
    return h


def test_reposing_and_export(seq, tmp_path):
    from selfreconcode_b200.avatar import TexturedAvatar, export_avatar, pose_vertices, rest_inverse
    net, ds, n = seq["net"], seq["net"].dataset, seq["n"]
    av = TexturedAvatar(seq["obj"], seq["tex"], DEV)
    ids = torch.arange(n)
    poses, trans, d_cond = ds.get_grad_parameters(ids, DEV)[:3]
    got = pose_vertices(net, av.V, poses, trans, d_cond)
    with torch.no_grad():
        want = net.deformer(av.V[None].expand(n, -1, 3), [d_cond, [poses, trans]],
                            ratio={'sdfRatio': 1., 'deformerRatio': 1., 'renderRatio': 1.})
    assert torch.equal(got, want)
    assert torch.equal(pose_vertices(net, av.V, poses.reshape(n, 72), trans, d_cond, np.zeros(n)), got)
    full = pose_vertices(net, av.V, poses, trans, d_cond, np.full(n, 360.)).cpu().numpy()
    turned = pose_vertices(net, av.V, poses, trans, d_cond, np.linspace(10., 300., n)).cpu().numpy()
    g0 = got.cpu().numpy().astype(np.float64)
    a = _turn_axis(ds)
    c = (net.deformer.defs[-1].Js[0].double().cpu().numpy()[None] + trans.double().cpu().numpy())[:, None]

    def dist(x):
        d = np.asarray(x, np.float64) - c
        return np.linalg.norm(d - (d @ a)[..., None] * a, axis=-1)
    e360 = np.abs(full - g0).max()
    eaxis = np.abs(dist(turned) - dist(g0)).max()
    moved = np.abs(turned - g0).max()
    # random poses with the code of frame 0 against translator + LBS in float64
    gen = torch.Generator().manual_seed(7)
    rp = (0.3 * torch.randn(5, 24, 3, generator=gen)).to(DEV)
    rt = (trans[:1].cpu() + 0.05 * torch.randn(5, 3, generator=gen)).to(DEV)
    code = d_cond[:1]
    posed = pose_vertices(net, av.V, rp, rt, code).cpu().numpy().astype(np.float64)
    tr, sk = net.deformer.defs[0], net.deformer.defs[-1]
    with torch.no_grad():
        q = av.V.double() + translator_f64(tr, av.V, code[0])
        g = 2. * (q - sk.b_min.double()) / (sk.b_max.double() - sk.b_min.double()) - 1.
        w = grid_sampler_ref.sample(sk.ws.double(), g.view(1, -1, 3))[0].t().cpu().numpy()
    rest = dict(Js=sk.Js.cpu().numpy(), parents=np.asarray([int(x) for x in sk.parents]),
                init_pose=rest_inverse(sk),
                skin_weights=w, verts=q.cpu().numpy())
    e_f64 = np.abs(posed - ref.lbs(rest, rp.cpu().numpy(), rt.cpu().numpy())).max()
    # the export
    path = str(tmp_path / "avatar.npz")
    export_avatar(net, av, path, cond_frame=0)
    z = np.load(path)
    assert str(z["texture"]) == "texture.png"
    assert z["skin_weights"].shape == (av.V.shape[0], 24) and z["init_pose"].shape == (24, 4, 4)
    assert np.array_equal(z["faces"], av.faces.cpu().numpy()) and np.array_equal(z["ft"], av.ft.cpu().numpy())
    e_exp = np.abs(ref.lbs(z, rp.cpu().numpy(), rt.cpu().numpy()) - posed).max()
    e_sum = np.abs(z["skin_weights"].astype(np.float64).sum(1) - 1.).max()
    print("reposing: yaw 360 max |d| %.2e, axis distances max |d| %.2e (moved up to %.3f); random poses vs float64 "
          "translator + LBS %.2e; export LBS %.2e, weight sums %.2e" % (e360, eaxis, moved, e_f64, e_exp, e_sum))
    assert e360 <= 1e-5 and eaxis <= 1e-5 and moved > 0.1
    assert e_f64 <= 2e-5
    assert e_exp <= 1e-5 and e_sum <= 1e-5


def test_outputs(seq, tmp_path):
    import cv2
    from selfreconcode_b200 import ops, synth
    from selfreconcode_b200.avatar import TexturedAvatar, pose_vertices, render_motion, render_sequence
    H.dropin()
    from model.raster import screen_vertices
    from model.CameraMine import RectifiedPerspectiveCameras
    net, ds, n, side = seq["net"], seq["net"].dataset, seq["n"], seq["side"]
    av = TexturedAvatar(seq["obj"], seq["tex"], DEV)
    out_dir = str(tmp_path / "seq")
    frames = [1, 4, 6]
    render_sequence(net, av, out_dir, frames=frames, batch=2)
    poses, trans, d_cond = ds.get_grad_parameters(torch.tensor(frames), DEV)[:3]
    D = pose_vertices(net, av.V, poses, trans, d_cond)
    f, pp, Rc, Tc, _, _ = ds.get_camera_parameters(len(frames), DEV)
    s = screen_vertices(D, RectifiedPerspectiveCameras(f, pp, Rc, Tc))
    cov = (ops.raster_mesh(s, av.faces, side, side)[0][..., 0] >= 0).cpu().numpy()
    lines = open(os.path.join(out_dir, "errors.txt")).read().splitlines()
    rows = [l for l in lines if l[:5].strip().rstrip(":").isdigit()]
    assert len(rows) == len(frames)
    mads = []
    for k, (fid, line) in enumerate(zip(frames, rows)):
        r = cv2.imread(os.path.join(out_dir, "%d.png" % fid)).astype(np.float64)
        fr = cv2.imread(ds.img_ns[fid]).astype(np.float64)
        m = cov[k] & (cv2.imread(ds.mask_ns[fid])[..., 0] > 0)
        d = np.abs(r - fr)[m]
        mad, psnr = d.mean(), 10 * np.log10(255. ** 2 / (d * d).mean())
        mads.append(mad)
        got = line.split(":")
        assert int(got[0]) == fid
        gm, gp = (float(x) for x in got[1].split())
        assert abs(gm - mad) <= 1e-4 and abs(gp - psnr) <= 1e-4, (fid, gm, mad, gp, psnr)
        # outside the render the frame shows through
        assert np.array_equal(r[~cov[k]], fr[~cov[k]])
    assert lines[-2].startswith("mad mean: %.4f, max: %.4f, min: %.4f" % (np.mean(mads), np.max(mads), np.min(mads)))
    cap = cv2.VideoCapture(os.path.join(out_dir, "video.mp4"))
    cnt = 0
    while cap.read()[0]:
        cnt += 1
    assert cnt == len(frames)
    # another sequence's motion, in the smpl_rec.npz layout
    T = 5
    p2, t2, _ = synth.make_frame_params(21, T)
    npz = str(tmp_path / "smpl_rec.npz")
    np.savez(npz, poses=p2.numpy().reshape(T, 72), trans=(t2 + seq["data"].trans[:1].detach().cpu()).numpy(),
             shape=np.zeros(10, np.float32))
    z = np.load(npz)
    mdir = str(tmp_path / "motion")
    render_motion(net, av, mdir, z["poses"], z["trans"], cond_frame=2, yaw_deg=np.linspace(0., 90., T), batch=2)
    imgs = [cv2.imread(os.path.join(mdir, "%d.png" % i)) for i in range(T)]
    assert all(im is not None and im.shape == (side, side, 3) for im in imgs)
    assert not os.path.exists(os.path.join(mdir, "%d.png" % T))
    white = np.all(imgs[0] == 255, -1)
    assert 0.2 < white.mean() < 0.99                      # the avatar over the white background
    cap = cv2.VideoCapture(os.path.join(mdir, "video.mp4"))
    cnt = 0
    while cap.read()[0]:
        cnt += 1
    assert cnt == T


def test_invalid_arguments():
    import ctypes as C
    from selfreconcode_b200 import _lib, ops
    lib = _lib.load()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.zeros(4096, device=DEV)
    p, z = C.c_void_p(buf.data_ptr()), C.c_void_p(0)
    mm = lib.sr_texture_mips
    assert mm(p, p, 4, 4, p, s) == 0
    for i in (0, 1, 4):
        a = [p, p, 4, 4, p, s]
        a[i] = z
        assert mm(*a) == _lib.SR_EINVAL, i
    for i in (2, 3):
        a = [p, p, 4, 4, p, s]
        a[i] = 0
        assert mm(*a) == _lib.SR_EINVAL, i
    assert mm(p, p, 4, 4, C.c_void_p(buf.data_ptr() + 4), s) == _lib.SR_EINVAL
    col = (C.c_float * 3)(1., 1., 1.)
    st = lib.sr_shade_textured
    ok = [p, p, 1, 2, 2, p, 3, p, p, 1, p, 3, p, 2, 2, z, col, p, s]
    for i in (0, 1, 5, 7, 8, 10, 12, 17):
        a = list(ok)
        a[i] = z
        assert st(*a) == _lib.SR_EINVAL, i
    a = list(ok)
    a[16] = None
    assert st(*a) == _lib.SR_EINVAL
    for i in (2, 3, 4, 6, 9, 11, 13, 14):
        a = list(ok)
        a[i] = 0
        assert st(*a) == _lib.SR_EINVAL, i
    a = list(ok)
    a[17] = C.c_void_p(buf.data_ptr() + 4)
    assert st(*a) == _lib.SR_EINVAL
    torch.cuda.synchronize()
    t8 = torch.zeros(4, 4, 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError):
        ops.texture_mips(t8.float(), torch.ones(4, 4, dtype=torch.bool, device=DEV))
    with pytest.raises(ValueError):
        ops.texture_mips(t8, torch.ones(4, 5, dtype=torch.bool, device=DEV))
    mips, levels = ops.texture_mips(t8, torch.ones(4, 4, dtype=torch.bool, device=DEV))
    p2f = torch.full((1, 2, 2), -1, dtype=torch.int64, device=DEV)
    args = [p2f, torch.zeros(1, 2, 2, 3, device=DEV), torch.ones(1, 3, 3, device=DEV),
            torch.tensor([[0, 1, 2]], device=DEV), torch.tensor([[0, 1, 2]], device=DEV), torch.rand(3, 2, device=DEV),
            mips, levels]
    out = ops.shade_textured(*args, background=(0.1, 0.2, 0.3))
    assert torch.equal(out, torch.tensor([0.1, 0.2, 0.3, 0.], device=DEV).expand(1, 2, 2, 4))
    with pytest.raises(ValueError):
        ops.shade_textured(*args, background=torch.zeros(1, 2, 2, 3, device=DEV))      # not uint8
    bad = list(args)
    bad[6] = mips[:-1]
    with pytest.raises(ValueError):
        ops.shade_textured(*bad)
    bad = list(args)
    bad[4] = torch.tensor([[0, 1]], device=DEV)
    with pytest.raises(ValueError):
        ops.shade_textured(*bad)
