"""GPU: the texture atlas (csrc/texture_bake.cu, selfreconcode_b200.texture) against the float64 restatement
(tests/texture_ref.py), a round trip through rendered frames, and bake_from_network end to end without pytorch3d /
opendr.  Scene: the synthetic template of test_gpu_mesh_shade._scene with two UV layouts, a chart per face pair and a
cylindrical layout whose faces share vertices (and seams)."""
import ctypes as C
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

import helpers as H
import raster_ref
import texture_ref as ref
from mesh_shade_ref import vertex_normals_p3d

pytestmark = pytest.mark.gpu
DEV = "cuda"


def chart_layout(F):
    """Every pair of faces gets one cell of an m x m grid (inset by 8 %), split along its diagonal."""
    m = int(math.ceil(math.sqrt((F + 1) // 2)))
    k = np.arange(F)
    cell = k // 2
    x0, y0 = (cell % m) / m, (cell // m) / m
    g, w = 0.08 / m, 1.0 / m
    a = np.stack([x0 + g, y0 + g], 1)
    b = np.stack([x0 + w - g, y0 + g], 1)
    c = np.stack([x0 + g, y0 + w - g], 1)
    d = np.stack([x0 + w - g, y0 + w - g], 1)
    odd = (k % 2 == 1)[:, None, None]
    tri = np.where(odd, np.stack([d, c, b], 1), np.stack([a, b, c], 1))
    return tri.reshape(-1, 2).astype(np.float32), np.arange(3 * F, dtype=np.int64).reshape(F, 3)


def seam_layout(verts, faces):
    """Cylindrical (u = angle about y, v = height) per vertex, so faces share their UV vertices; a face across the
    seam takes copies of its low-u vertices shifted by one turn (partly off the atlas).  Near the poles the map folds,
    so some UV faces overlap there."""
    v = np.asarray(verts, np.float64)
    u = 0.05 + 0.9 * (np.arctan2(v[:, 0], v[:, 2]) / (2 * np.pi) + 0.5)
    h = (v[:, 1] - v[:, 1].min()) / (v[:, 1].max() - v[:, 1].min())
    vt = np.stack([u, 0.05 + 0.9 * h], 1)
    ft = np.asarray(faces, np.int64).copy()
    fu = u[ft]
    wrap = (fu.max(1) - fu.min(1) > 0.45)[:, None] & (fu < 0.5)
    ft[wrap] += v.shape[0]
    return np.concatenate([vt, vt + [0.9, 0.]]).astype(np.float32), ft


_SCENES = {}


def scene(side, n_frames):
    """(net, data, cams, TmpVs, Tmpfs) with per-frame root rotations of +-0.6 rad about y on top of the poses."""
    key = (side, n_frames)
    if key not in _SCENES:
        from test_gpu_mesh_shade import _scene
        net, data, cams, TmpVs, Tmpfs, _ = _scene(side, side, n_frames)
        with torch.no_grad():
            data.poses[:, 0, 1] = torch.linspace(-0.6, 0.6, n_frames, device=data.poses.device)
        _SCENES[key] = (net, data, cams, TmpVs, Tmpfs.long())
    return _SCENES[key]


def deformed(net, data, TmpVs, ids):
    poses, trans, d_cond, _ = data.get_grad_parameters(torch.as_tensor(ids, device=DEV), DEV)
    with torch.no_grad():
        return net.deformer(TmpVs[None].expand(len(ids), -1, 3), [d_cond, [poses, trans]], ratio=H.RATIO)


def layout(name, TmpVs, Tmpfs):
    if name == "chart":
        return chart_layout(Tmpfs.shape[0])
    return seam_layout(TmpVs.cpu().numpy(), Tmpfs.cpu().numpy())


def baker_for(Tmpfs, vt, ft, R, S=50, min_views=5):
    from selfreconcode_b200.texture import TextureBaker
    return TextureBaker(Tmpfs, torch.from_numpy(vt), torch.from_numpy(ft), R, S, 68., min_views, DEV)


def texel_faces(baker):
    R = baker.R
    face = -np.ones(R * R, np.int64)
    bary = np.zeros((R * R, 3))
    idx = baker.texel_index.cpu().numpy()
    face[idx] = baker.texel_face.cpu().numpy()
    bary[idx] = baker.texel_bary.cpu().numpy()
    return face.reshape(R, R), bary.reshape(R, R, 3)


# ---- 1. UV raster -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,R", [("chart", 1024), ("seam", 512)])
def test_uv_raster_vs_restatement(name, R):
    _, _, _, TmpVs, Tmpfs = scene(96, 2)
    vt, ft = layout(name, TmpVs, Tmpfs)
    baker = baker_for(Tmpfs, vt, ft, R, S=2, min_views=1)
    got_f, got_b = texel_faces(baker)
    want_f, want_b, near, overlap = ref.uv_raster(ref.uv_screen(vt, R), ft, R)
    # the rasteriser's restatement on the same atlas vertices at depth 1: a texel may go to either face only where the
    # choice is sensitive to fp32 rounding (near an edge, or inside overlapping faces whose depths tie), and may be
    # left empty only on an outline (never near an edge shared by faces on opposite sides of it)
    xy = ref.uv_screen(vt, R)
    rr = raster_ref.raster(np.concatenate([xy, np.ones((xy.shape[0], 1))], 1)[None], ft, R, R)
    sens, must, outline = rr.sensitive[0], rr.must_cover[0], rr.outline[0]
    diff = got_f != want_f
    same = (got_f >= 0) & ~diff
    berr = float(np.abs(got_b - want_b)[same].max())
    holes = (got_f < 0) & (want_f >= 0)
    print("UV raster %s R=%d: %d covered texels; %d sensitive, %d differ there; %d must-cover, %d empty there; %d outline, "
          "%d empty there; %d differ elsewhere; %d inside two overlapping faces; barycentrics max |err| %.2e"
          % (name, R, (want_f >= 0).sum(), sens.sum(), (diff & sens).sum(), must.sum(), (must & (got_f < 0)).sum(),
             outline.sum(), (holes & outline).sum(), (diff & ~sens).sum(), overlap.sum(), berr))
    assert (want_f >= 0).sum() > 0.3 * R * R
    assert not (diff & ~sens).any()
    assert not (must & (got_f < 0)).any() and not (holes & ~outline).any()
    assert (got_f >= 0)[overlap].all() and overlap.sum() < (0.02 * R * R if name == "seam" else 1)
    assert berr <= 1e-4
    assert torch.equal(baker.tex_mask.cpu(), torch.from_numpy(got_f >= 0))


# ---- 2. accumulate + finish ---------------------------------------------------------------------------------------
def smooth_image(n, side):
    yy, xx = np.meshgrid(np.arange(side, dtype=np.float64), np.arange(side, dtype=np.float64), indexing="ij")
    chans = [127.5 + 100. * np.sin(xx / (13. + c) + 0.7 * n + c) * np.cos(yy / (17. - 2 * c) - 0.3 * n) for c in range(3)]
    return np.clip(np.rint(np.stack(chans, -1)), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("name,R,S,min_views", [("chart", 1024, 8, 3), ("seam", 512, 50, 5)])
def test_accumulate_finish_vs_restatement(name, R, S, min_views):
    from selfreconcode_b200 import ops
    H.dropin()
    from model.raster import screen_vertices
    n_frames, side = 12, 256
    net, data, cams, TmpVs, Tmpfs = scene(side, n_frames)
    vt, ft = layout(name, TmpVs, Tmpfs)
    baker = baker_for(Tmpfs, vt, ft, R, S, min_views)
    D = deformed(net, data, TmpVs, list(range(n_frames)))
    T = baker.texel_index.numel()
    slots = ref.Slots(T, S, baker.c0)
    tf, tb = baker.texel_face.cpu().numpy(), baker.texel_bary.cpu().numpy()
    fc = Tmpfs.cpu().numpy()
    cam_pos = cams.cam_pos(0).double().cpu().numpy()
    a_err = 0.
    for n in range(n_frames):
        img = smooth_image(n, side)
        cov = ops.raster_mesh(screen_vertices(D[n:n + 1], cams), Tmpfs, side, side)[0][0, ..., 0].cpu().numpy() >= 0
        mask = cov & (np.arange(side)[None, :] < 0.8 * side)          # part of the body is outside the mask
        screen, weight, usable = baker.frame_inputs(D[n], cams, torch.from_numpy(mask))
        # the per-vertex / per-face inputs against their rule
        s = screen.cpu().numpy().astype(np.float64)
        p2f = ops.raster_mesh(screen[None], Tmpfs, side, side)[0].view(-1).cpu().numpy()
        owned = np.zeros(fc.shape[0], bool)
        owned[p2f[p2f >= 0]] = True
        want_usable = ref.vertex_in_mask(s, mask)[fc].all(1) & owned
        assert np.array_equal(usable.cpu().numpy() > 0, want_usable)
        dv = D[n].double().cpu().numpy()
        nr = vertex_normals_p3d(dv[None], fc)[0]
        dirs = dv - cam_pos
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        a_err = max(a_err, float(np.abs(weight.cpu().numpy() - np.maximum(0., -(nr * dirs).sum(1))).max()))
        fid = 3 * n + 1
        baker.accumulate(screen, weight, usable, torch.from_numpy(img).to(DEV), fid)
        ref.accumulate(slots, tf, tb, s, fc, weight.cpu().numpy(), usable.cpu().numpy(), img, fid)
    out = baker.finish()
    out2 = baker.finish()
    for k in ("tex_median", "view_id", "count", "mask_final"):
        assert torch.equal(out[k], out2[k]), k
    med, mf, view, count = ref.finish(slots, min_views)
    idx = baker.texel_index.cpu().numpy()
    g = {k: out[k].reshape(R * R, -1).cpu().numpy()[idx] for k in out}
    keep = ~slots.close
    d_count = int((g["count"][:, 0] != count)[keep].sum())
    d_mask = int((g["mask_final"][:, 0] != mf)[keep].sum())
    d_view = int((g["view_id"][:, 0] != view)[keep].sum())
    both = keep & mf & g["mask_final"][:, 0]
    m_err = float(np.abs(g["tex_median"] - med)[both].max())
    print("accumulate/finish %s R=%d S=%d: %d texels, %d final, %d with all %d slots filled; %d excluded (alpha within "
          "1e-6 of a compared slot); count/mask/view differences %d/%d/%d; tex_median max |err| %.2e; a_v max |err| %.1e"
          % (name, R, S, T, mf.sum(), (count == S).sum(), S, (~keep).sum(), d_count, d_mask, d_view, m_err, a_err))
    assert d_count == 0 and d_mask == 0 and d_view == 0
    assert m_err <= 1e-4 and a_err <= 1e-5
    assert mf.sum() > 0.05 * T and (~keep).sum() < 0.01 * T
    if S < n_frames:
        assert (count == S).sum() > 1000          # slots filled up and were replaced
    untouched = ~out["tex_mask"].cpu().numpy()
    assert (out["view_id"].cpu().numpy()[untouched] == -1).all() and (out["count"].cpu().numpy()[untouched] == 0).all()


# ---- 3. round trip ------------------------------------------------------------------------------------------------
G_A = np.array([[20., 9., 5.], [-7., 18., 11.], [12., -6., 19.]])
G_PHI = np.array([0.3, 1.9, 4.1])


def g_colour(x):
    """Smooth colour of a canonical point, [..., 3] in [0.1, 0.9]."""
    return 0.5 + 0.4 * np.sin(np.asarray(x, np.float64) @ G_A.T + G_PHI)


def test_round_trip():
    """Frames rendered with pixel colour g(canonical point seen there) on the deformed template (the body), a small
    copy of it fixed between the camera and the body (inside the mask: it hides the body's centre in every frame) and a
    second copy beside the body painted magenta and left out of the mask.  The baked median must equal g at every
    texel's canonical point wherever mask_final is set; without the visibility test, without the mask test, or with
    the image sampled half a pixel off, it must not."""
    from selfreconcode_b200 import ops
    H.dropin()
    from model.raster import screen_vertices
    n_frames, side, R = 24, 384, 1536
    net, data, cams, TmpVs, Tmpfs = scene(side, n_frames)
    V, F = TmpVs.shape[0], Tmpfs.shape[0]
    faces = torch.cat([Tmpfs, Tmpfs + V, Tmpfs + 2 * V])
    canon = torch.cat([TmpVs, 0.3 * TmpVs + torch.tensor([3., 0., 0.], device=DEV),
                       0.2 * TmpVs + torch.tensor([-3., 0., 0.], device=DEV)])
    vt, ft = chart_layout(3 * F)
    bakers = {k: baker_for(faces, vt, ft, R) for k in ("rule", "no visibility", "no mask", "half pixel")}
    body = deformed(net, data, TmpVs, list(range(n_frames)))
    prop = 0.2 * TmpVs + torch.tensor([1.0, 0.3, 2.5], device=DEV)
    cn = canon.double().cpu().numpy()
    fc = faces.cpu().numpy()
    for n in range(n_frames):
        # the occluder circles in front of the body's centre while the body turns: the body's centre is behind it in
        # most frames, and no texel lies on its outline in most of the frames that see it
        # and turns, so that its own outline moves over its surface as the body's does
        th = 2 * math.pi * 5 * n / n_frames
        a, b = 0.6 * math.sin(2 * math.pi * 3 * n / n_frames), 0.4 * math.cos(2 * math.pi * 2 * n / n_frames)
        ry = torch.tensor([[math.cos(a), 0., math.sin(a)], [0., 1., 0.], [-math.sin(a), 0., math.cos(a)]])
        rx = torch.tensor([[1., 0., 0.], [0., math.cos(b), -math.sin(b)], [0., math.sin(b), math.cos(b)]])
        occl = 0.3 * TmpVs @ (rx @ ry).T.to(DEV) + torch.tensor([0.12 * math.cos(th), 0.05 + 0.12 * math.sin(th), 1.7],
                                                                device=DEV)
        D = torch.cat([body[n], occl, prop]).contiguous()
        s = screen_vertices(D[None], cams)
        p2f, bary, _ = ops.raster_mesh(s, faces, side, side)
        p2f, bary = p2f[0, ..., 0].cpu().numpy(), bary[0, ..., 0, :].cpu().numpy().astype(np.float64)
        hit = p2f >= 0
        col = np.zeros((side, side, 3))
        col[hit] = g_colour((bary[hit][:, :, None] * cn[fc[p2f[hit]]]).sum(1))
        in_prop = hit & (p2f >= 2 * F)
        col[in_prop] = [1., 0., 1.]
        img = torch.from_numpy(np.rint(col * 255.).astype(np.uint8)).to(DEV)
        mask = torch.from_numpy(hit & ~in_prop)
        assert in_prop.sum() > 100 and (p2f[hit] >= F).sum() > 1000
        screen, weight, usable = bakers["rule"].frame_inputs(D, cams, mask)
        sc = screen.cpu().numpy().astype(np.float64)
        in_mask_faces = torch.from_numpy(ref.vertex_in_mask(sc, mask.numpy())[fc].all(1)).to(DEV)
        owned = torch.zeros(3 * F, dtype=torch.bool, device=DEV)
        owned[torch.from_numpy(p2f[hit]).to(DEV)] = True     # the render is this frame's raster of the same mesh
        u8 = lambda b: b.to(torch.uint8)
        assert torch.equal(usable, u8(in_mask_faces & owned))
        bakers["rule"].accumulate(screen, weight, usable, img, n)
        bakers["no visibility"].accumulate(screen, weight, u8(in_mask_faces), img, n)
        bakers["no mask"].accumulate(screen, weight, u8(owned), img, n)
        bakers["half pixel"].accumulate(screen + torch.tensor([0.5, 0.5, 0.], device=DEV), weight, usable, img, n)
    errs = {}
    for k, b in bakers.items():
        out = b.finish()
        tf, tb = b.texel_face.cpu().numpy(), b.texel_bary.cpu().numpy().astype(np.float64)
        want = g_colour((tb[:, :, None] * cn[fc[tf]]).sum(1))
        idx = b.texel_index.cpu().numpy()
        mf = out["mask_final"].view(-1).cpu().numpy()[idx]
        got = out["tex_median"].view(-1, 3).cpu().numpy()[idx].astype(np.float64)
        e = np.abs(got - want).max(1)[mf]
        part = np.where(tf < F, 0, np.where(tf < 2 * F, 1, 2))[mf]
        errs[k] = (np.quantile(e, 0.99), (e > 4. / 255.).mean())
        print("round trip (%s): %d texels final (body %d, occluder %d, prop %d); |err| max %.2f/255, p99.99 %.2f/255, "
              "p99.9 %.2f/255, p99 %.2f/255, mean %.3f/255; above 4/255: %d body, %d occluder, %d prop"
              % (k, mf.sum(), (part == 0).sum(), (part == 1).sum(), (part == 2).sum(), 255 * e.max(),
                 255 * np.quantile(e, 0.9999), 255 * np.quantile(e, 0.999), 255 * np.quantile(e, 0.99), 255 * e.mean(),
                 ((e > 4 / 255) & (part == 0)).sum(),
                 ((e > 4 / 255) & (part == 1)).sum(), ((e > 4 / 255) & (part == 2)).sum()))
        if k == "rule":
            assert (part == 0).sum() > 20000 and (part == 1).sum() > 2000 and (part == 2).sum() == 0
            # the body's centre, behind the occluder in every frame, is never seen
            body_tex = tf < F
            assert (mf[body_tex] == 0).sum() > 1000
    # Bars from measurement (one H100): p99 1.18/255, 0.15 % of the final texels above 4/255.  Those few lie at an
    # outline in most of the views they keep (a face at the outline owns a pixel, or the bilinear footprint crosses
    # it): the rule's own behaviour, so the maximum (79/255) is not a bar; the device's own error is bounded by
    # test_accumulate_finish_vs_restatement.
    p99, frac = errs["rule"]
    assert p99 <= 2. / 255. and frac <= 0.005
    for k in ("no visibility", "no mask", "half pixel"):
        assert errs[k][0] > 4. / 255. and errs[k][1] > 0.02, k


# ---- 4. bake_from_network -----------------------------------------------------------------------------------------
def write_obj(path, V, F, vt, ft):
    with open(path, "w") as fh:
        fh.write("".join("v %.9g %.9g %.9g\n" % tuple(p) for p in V))
        fh.write("".join("vt %.9g %.9g\n" % tuple(p) for p in vt))
        fh.write("".join("f %d/%d %d/%d %d/%d\n" % (a + 1, x + 1, b + 1, y + 1, c + 1, z + 1)
                         for (a, b, c), (x, y, z) in zip(F, ft)))


def test_bake_from_network(tmp_path, monkeypatch):
    import cv2
    from selfreconcode_b200 import ops
    from selfreconcode_b200.texture import bake_from_network, load_obj_uv
    H.dropin()
    from dataset import write_sequence
    from dataset.dataset import SceneDataset
    from model.raster import screen_vertices
    n_frames, side, R = 6, 160, 256
    net, data, cams, TmpVs, Tmpfs = scene(side, n_frames)
    vt, ft = chart_layout(Tmpfs.shape[0])
    obj = str(tmp_path / "uvmap.obj")
    write_obj(obj, TmpVs.cpu().numpy(), Tmpfs.cpu().numpy(), vt, ft)
    Vr = load_obj_uv(obj)[0]
    D = deformed(net, data, Vr.to(DEV), list(range(n_frames)))
    imgs, masks = [], []
    for n in range(n_frames):
        p2f, bary, _ = ops.raster_mesh(screen_vertices(D[n:n + 1], cams), Tmpfs, side, side)
        hit = p2f[0, ..., 0].cpu().numpy() >= 0
        imgs.append(np.where(hit[..., None], smooth_image(n, side), 0).astype(np.float32) / 255. * 2 - 1)
        masks.append(hit.astype(np.float32))
    root = str(tmp_path / "seq")
    f, pp = data.focals.detach().view(2).cpu().numpy(), data.pps.detach().view(2).cpu().numpy()
    write_sequence(root, np.stack(imgs), np.stack(masks), data.poses.detach().cpu().numpy(),
                   data.trans.detach().cpu().numpy(), np.zeros(10, np.float32),
                   dict(fx=f[0], fy=f[1], cx=pp[0], cy=pp[1], quat=[0., 0., 0., 1.], T=[0., 0., 0.]))
    ds = SceneDataset(root, {'deformer': 128})
    with torch.no_grad():
        ds.conds[0].copy_(data.conds[0].detach().cpu())
    # what bake_from_network reads of optNet (the test's network holds its synthetic dataset as a child module)
    net = types.SimpleNamespace(deformer=net.deformer, dataset=ds)
    monkeypatch.setitem(sys.modules, "pytorch3d", None)
    monkeypatch.setitem(sys.modules, "opendr", None)
    with pytest.raises(ImportError):
        import pytorch3d  # noqa: F401
    outs = []
    for run in range(2):
        out_dir = str(tmp_path / ("tex%d" % run))
        outs.append(bake_from_network(net, obj, out_dir, num=n_frames, resolution=R, min_views=2))
        for png in ("tex_mask", "mask_final", "tex_median", "texture"):
            im = cv2.imread(os.path.join(out_dir, png + ".png"), cv2.IMREAD_UNCHANGED)
            assert im is not None and im.shape[:2] == (R, R), png
        med = cv2.imread(os.path.join(out_dir, "tex_median.png"))
        assert np.array_equal(med, np.uint8(outs[-1]["tex_median"].cpu().numpy().astype(np.float64) * 255))
    assert torch.equal(outs[0]["tex_median"], outs[1]["tex_median"]) and torch.equal(outs[0]["view_id"], outs[1]["view_id"])
    mf = outs[0]["mask_final"].cpu().numpy()
    print("bake_from_network: %d frames %dx%d, atlas %d^2, %d texels final" % (n_frames, side, side, R, mf.sum()))
    assert mf.sum() > 1000 and set(np.unique(outs[0]["view_id"].cpu().numpy())) <= set(range(-1, n_frames))
    # a frame file whose number is not the frame id
    ds.img_ns = ds.img_ns[1:] + ds.img_ns[:1]
    with pytest.raises(ValueError):
        bake_from_network(net, obj, str(tmp_path / "bad"), num=n_frames, resolution=R, min_views=2)


# ---- 5. invalid arguments -----------------------------------------------------------------------------------------
def test_invalid_arguments():
    from selfreconcode_b200 import _lib
    from selfreconcode_b200.texture import TextureBaker, texture_frame_ids
    lib = _lib.load()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.zeros(4096, device=DEV)
    p = C.c_void_p(buf.data_ptr())
    z = C.c_void_p(0)
    acc = lib.sr_texture_accumulate
    ok = [4, 2, p, p, p, p, 3, 1, p, p, p, 4, 4, 0, p, p, p, p, p, s]
    for i in (2, 3, 4, 5, 8, 9, 10, 14, 15, 16, 17, 18):
        a = list(ok)
        a[i] = z
        assert acc(*a) == _lib.SR_EINVAL, i
    for i, bad in ((0, 0), (1, 0), (1, 65), (6, 0), (7, 0), (11, 0), (12, -1), (13, -1)):
        a = list(ok)
        a[i] = bad
        assert acc(*a) == _lib.SR_EINVAL, i
    fin = lib.sr_texture_finish
    ok = [4, 2, p, p, p, p, 0.5, 1, p, p, p, p, s]
    for i in (2, 3, 4, 5, 8, 9, 10, 11):
        a = list(ok)
        a[i] = z
        assert fin(*a) == _lib.SR_EINVAL, i
    for i, bad in ((0, 0), (1, 0), (1, 65), (6, 0.), (6, 1.), (7, 0), (7, 3)):
        a = list(ok)
        a[i] = bad
        assert fin(*a) == _lib.SR_EINVAL, i
    torch.cuda.synchronize()
    vt = torch.tensor([[0., 0.], [1., 0.], [0., 1.]])
    f = torch.tensor([[0, 1, 2]])
    for kw in (dict(max_angle=0.), dict(max_angle=90.), dict(max_angle=-5.), dict(min_views=0),
               dict(min_views=51), dict(resolution=0), dict(views=0), dict(views=65, min_views=5)):
        args = dict(resolution=8, views=50, max_angle=68., min_views=5)
        args.update(kw)
        with pytest.raises(ValueError):
            TextureBaker(f, vt, f, device=DEV, **args)
    with pytest.raises(ValueError):
        TextureBaker(f, vt, torch.tensor([[0, 1, 2], [0, 1, 2]]), resolution=8, device=DEV)
    with pytest.raises(ValueError):
        texture_frame_ids(121, 120)
    b = TextureBaker(f, vt, f, resolution=8, views=4, min_views=2, device=DEV)
    with pytest.raises(ValueError):
        b.add_frame(torch.zeros(3, 3, device=DEV), None, np.zeros((4, 4, 3), np.uint8), np.zeros((4, 4), bool), -1)
    with pytest.raises(ValueError):
        b.add_frame(torch.zeros(3, 3, device=DEV), None, np.zeros((4, 4), np.uint8), np.zeros((4, 4), bool), 0)
