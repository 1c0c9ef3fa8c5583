"""GPU: the device vertex normals and Phong shader (csrc/mesh_shade.cu) against the float64 restatement of pytorch3d's
rules (tests/mesh_shade_ref.py), and OptimNetwork.infer end to end on the built-in renderer with pytorch3d unimportable.

Bars: vertex normals |a-b| <= 1e-5 per component, shaded RGB <= 2e-5 absolute, background / alpha / back-lit pixels
exact; infer's images within 1 LSB of the test's own composition (rasteriser + restated shading + clamp * 255)."""
import ctypes as C
import sys

import numpy as np
import pytest
import torch

import helpers as H
from mesh_shade_ref import shade_phong_p3d, vertex_normals_p3d

pytestmark = pytest.mark.gpu
DEV = "cuda"


def mc_mesh():
    """Marching-cubes mesh of a bumpy sphere, plus zero-area faces and one unreferenced vertex."""
    from selfreconcode_b200 import ops
    zz, yy, xx = torch.meshgrid([torch.linspace(-1, 1, 41)] * 3, indexing="ij")
    grid = (torch.sqrt(xx * xx + yy * yy + zz * zz) - 0.6 + 0.05 * torch.sin(5 * xx) * torch.cos(3 * yy)).contiguous()
    v, f = ops.marching_cubes(grid.to(DEV), 0.05, 0.05, 0.05, -1.0, -1.0, -1.0, 0.0)
    v, f = v.float(), f.long()
    V = v.shape[0]
    a, b = f[0, 0], f[0, 1]
    mid = 0.5 * (v[a] + v[b])                                   # vertex V: on the edge (a, b)
    v = torch.cat([v, mid.view(1, 3), torch.tensor([[2., 2., 2.]], device=DEV)])   # vertex V+1: unreferenced
    extra = torch.tensor([[a, a, b], [a, b, V], [b, b, b], [f[5, 0], f[5, 2], f[5, 2]]], device=DEV)
    return v.contiguous(), torch.cat([f, extra]).contiguous(), V + 1


def frames(v, n=3):
    out = []
    for k in range(n):
        s = 1.0 + 0.1 * k
        w = v * torch.tensor([s, 1.0 / s, 1.0], device=DEV) + 0.08 * torch.sin((2.0 + k) * v[:, [1, 2, 0]] + k)
        out.append(w)
    return torch.stack(out).contiguous()


def csr_of(faces, V):
    H.dropin()
    from model.raster import vertex_face_csr
    return vertex_face_csr(faces, V)


def test_vertex_normals_vs_restatement():
    from selfreconcode_b200 import ops
    v, f, unref = mc_mesh()
    vs = frames(v)
    csr = csr_of(f, v.shape[0])
    assert int(csr[0][-1]) == 3 * f.shape[0] and torch.all(csr[0][1:] >= csr[0][:-1])
    n1 = ops.mesh_vertex_normals(vs, f, csr)
    n2 = ops.mesh_vertex_normals(vs, f, csr)
    torch.cuda.synchronize()
    assert torch.equal(n1, n2), "reruns must be bit-identical"
    got = n1.cpu().numpy()
    ref = vertex_normals_p3d(vs.cpu().numpy(), f.cpu().numpy())
    err = np.abs(got - ref).max()
    print("vertex normals: %d frames x %d vertices, %d faces, max |err| %.2e" % (vs.shape[0], v.shape[0], f.shape[0], err))
    assert err <= 1e-5
    assert np.array_equal(got[:, unref], np.zeros((vs.shape[0], 3)))
    # negative control: the openmesh rule (unit face normals) is a different function
    ctl = np.abs(got - vertex_normals_p3d(vs.cpu().numpy(), f.cpu().numpy(), unit_faces=True)).max()
    print("   unit-face-normal control: max |err| %.2e" % ctl)
    assert ctl > 1e-5


def _cameras(Hh, Ww):
    H.dropin()
    from model.CameraMine import RectifiedPerspectiveCameras
    c, s = np.cos(np.radians(30.)), np.sin(np.radians(30.))
    R0 = torch.diag(torch.tensor([-1., -1., 1.]))
    Ry = torch.tensor([[c, 0., s], [0., 1., 0.], [-s, 0., c]], dtype=torch.float32)
    R = torch.stack([R0, Ry @ R0])
    T = torch.tensor([[0., 0., 2.5], [0.05, -0.02, 2.6]])
    focal = torch.tensor([[float(Ww), float(Ww)], [1.1 * Ww, 1.05 * Ww]])
    pp = torch.tensor([[Ww / 2.0, Hh / 2.0], [Ww / 2.0 + 3.0, Hh / 2.0 - 2.0]])
    return RectifiedPerspectiveCameras(focal, pp, R, T, image_size=[(Ww, Hh)]).to(DEV)


def _cam_pos(cams, N):
    return np.stack([cams.cam_pos(n).double().cpu().numpy() for n in range(N)])


LIGHTS = [[-1.0, 1.5, -1.5], [0.8, 0.6, -2.0]]


@pytest.mark.parametrize("with_colors", [False, True])
def test_shading_vs_restatement(with_colors):
    H.dropin()
    from model.raster import (HardPhongShader, MeshRasterizer, MeshRenderer, PointLights, RasterSettings,
                              SilhouetteRenderer)
    v, f, _ = mc_mesh()
    vs = frames(v, 2)
    Hh, Ww = 120, 136
    cams = _cameras(Hh, Ww)
    ras = MeshRasterizer(cams, RasterSettings((Hh, Ww)))
    lights = PointLights(device=DEV, location=LIGHTS)
    rend = MeshRenderer(ras, HardPhongShader(DEV, cams, lights=lights))
    cols = None
    if with_colors:
        g = torch.Generator().manual_seed(4)
        cols = torch.rand(vs.shape, generator=g).to(DEV)
    img, frags = rend(vs, f, verts_colors=cols)
    torch.cuda.synchronize()
    _, sfr = SilhouetteRenderer(ras)(vs, f)
    for k in ("pix_to_face", "bary_coords", "zbuf"):
        assert torch.equal(getattr(frags, k), getattr(sfr, k)), k
    p2f = frags.pix_to_face[..., 0].cpu().numpy()
    bary = frags.bary_coords[..., 0, :].cpu().numpy()
    vn = vertex_normals_p3d(vs.cpu().numpy(), f.cpu().numpy())
    cp = _cam_pos(cams, 2)
    args = (vs.cpu().numpy(), vn, f.cpu().numpy(), p2f, bary, cp)
    ck = dict(colors=None if cols is None else cols.cpu().numpy())
    ref, terms = shade_phong_p3d(*args, np.array(LIGHTS), **ck)
    got = img.cpu().numpy()
    cov = p2f >= 0
    assert cov[0].sum() > 2000 and cov[1].sum() > 2000
    err = np.abs(got[..., :3] - ref[..., :3])[cov].max()
    print("shading (colours %s): %d covered pixels, max |rgb err| %.2e, highlight max %.3f"
          % (with_colors, cov.sum(), err, terms["specular"].max()))
    assert err <= 2e-5
    assert np.array_equal(got[~cov], np.tile(np.float32([1, 1, 1, 0]), ((~cov).sum(), 1)))
    assert np.all(got[..., 3][cov] == 1.0)
    back = cov & (terms["cos"] < -1e-6)
    assert back.sum() > 100
    if cols is None:      # ambient only: exactly 0.5 (no diffuse, no specular)
        assert np.all(got[back][:, :3] == 0.5)
    else:                 # the restatement is 0.5 * texel there
        assert np.abs(got[back][:, :3] - ref[back][:, :3]).max() <= 1e-6
    # negative controls: no specular term; the light fixed at (0, 1, 0) instead of per frame
    ctl1 = np.abs(got[..., :3] - shade_phong_p3d(*args, np.array(LIGHTS), specular=False, **ck)[0][..., :3])[cov].max()
    ctl2 = np.abs(got[..., :3] - shade_phong_p3d(*args, np.array([[0., 1., 0.]] * 2), **ck)[0][..., :3])[cov].max()
    print("   controls: without specular %.2e, fixed light %.2e" % (ctl1, ctl2))
    assert ctl1 > 2e-5 and ctl2 > 2e-5


def test_invalid_arguments():
    from selfreconcode_b200 import _lib
    lib = _lib.load()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.zeros(4096, device=DEV)
    p = C.c_void_p(buf.data_ptr())
    z = C.c_void_p(0)
    prm = _lib.PhongParams()
    vn = lib.sr_mesh_vertex_normals
    assert vn(z, p, p, p, 1, 3, 1, p, s) == _lib.SR_EINVAL
    assert vn(p, p, z, p, 1, 3, 1, p, s) == _lib.SR_EINVAL
    assert vn(p, p, p, p, 0, 3, 1, p, s) == _lib.SR_EINVAL
    assert vn(p, p, p, p, 1, 0, 1, p, s) == _lib.SR_EINVAL
    assert vn(p, p, p, p, 1, 3, -1, p, s) == _lib.SR_EINVAL
    sp = lib.sr_shade_phong
    ok = [p, p, z, p, 1, 3, 1, p, p, 4, 4, p, p, C.byref(prm), p, s]
    for i in (0, 1, 3, 7, 8, 11, 12, 14):
        a = list(ok)
        a[i] = z
        assert sp(*a) == _lib.SR_EINVAL, i
    a = list(ok)
    a[13] = None
    assert sp(*a) == _lib.SR_EINVAL
    for i, bad in ((4, 0), (5, 0), (6, 0), (9, 0), (10, -1)):
        a = list(ok)
        a[i] = bad
        assert sp(*a) == _lib.SR_EINVAL, i
    a = list(ok)
    a[14] = C.c_void_p(buf.data_ptr() + 4)       # float4 stores need a 16-byte aligned output
    assert sp(*a) == _lib.SR_EINVAL
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# OptimNetwork.infer end to end
# ---------------------------------------------------------------------------------------------------------------------
def _scene(Hh=112, Ww=96, n_frames=2):
    H.dropin()
    from selfreconcode_b200 import synth
    from model.Deformer import CompositeDeformer
    from model.optim import OptimNetwork
    from model.CameraMine import RectifiedPerspectiveCameras
    from model.raster import MeshRasterizer, RasterSettings, SilhouetteRenderer
    from MCAcc import Seg3dLossless
    sdf = synth.make_sdf().to(DEV)
    comp = CompositeDeformer([synth.make_translator(), synth.make_skinner(resolution=(33, 57, 17))]).to(DEV)
    rn = synth.make_render().to(DEV)
    data = synth.SyntheticDataset(n_frames, Hh, Ww).to(DEV)
    with torch.no_grad():
        # the body 2.5 in front of a camera at the origin (same view as synth.camera), so that the front camera of
        # def1imgs (T = mean translation, network.py:336-337) sees the canonical template from outside
        data.trans[:, 2] += 2.5
        data.Ts.zero_()
    f, pp, R, T, _, _ = data.get_camera_parameters(n_frames, DEV)
    cams = RectifiedPerspectiveCameras(f.detach(), pp.detach(), R, T.detach(), image_size=[(Ww, Hh)])
    eng = Seg3dLossless(query_func=None, b_min=[-0.9, -0.9, -0.9], b_max=[0.9, 0.9, 0.9],
                        resolutions=[(9, 9, 9), (17, 17, 17), (33, 33, 33), (65, 65, 65)],
                        align_corners=False, balance_value=0.0, use_cuda_impl=True).to(DEV)
    net = OptimNetwork(sdf, comp, eng, SilhouetteRenderer(MeshRasterizer(cams, RasterSettings((Hh, Ww)))), rn,
                       conf=synth.Conf(grad_weight=0.1))
    net.dataset = data
    TmpVs, Tmpfs = net.discretizeSDF(H.RATIO, None, 0.0)
    return net, data, cams, TmpVs.detach(), Tmpfs, torch.arange(n_frames, device=DEV)


def _recording(base_cls):
    class Recording(base_cls):
        def __init__(self, *a):
            super().__init__(*a)
            self.calls = []

        def __call__(self, verts, faces, cameras=None, lights=None, **kw):
            img, frags = super().__call__(verts, faces, cameras=cameras, lights=lights, **kw)
            self.calls.append(dict(verts=verts.detach().clone(), cameras=cameras, lights=lights, frags=frags))
            return img, frags
    return Recording


def _gts(N, Hh, Ww, image):
    yy, xx = torch.meshgrid(torch.arange(Hh, device=DEV).float(), torch.arange(Ww, device=DEV).float(), indexing="ij")
    m = (((yy - Hh / 2) / (0.3 * Hh)) ** 2 + ((xx - Ww / 2) / (0.25 * Ww)) ** 2 < 1).float()
    g = {'mask': m.expand(N, Hh, Ww).contiguous()}
    if image:
        gen = torch.Generator().manual_seed(11)
        g['image'] = torch.rand(N, Hh, Ww, 3, generator=gen).to(DEV)
    return g


def _composed(call, faces, cam_pos, light, channels):
    p2f = call["frags"].pix_to_face[..., 0].cpu().numpy()
    bary = call["frags"].bary_coords[..., 0, :].cpu().numpy()
    vs = call["verts"].cpu().numpy()
    ref, _ = shade_phong_p3d(vs, vertex_normals_p3d(vs, faces), faces, p2f, bary, cam_pos,
                             np.broadcast_to(np.asarray(light, np.float64), cam_pos.shape))
    return np.clip(ref[..., :channels] * 255., 0., 255.).astype(np.uint8)


def test_infer_builtin_renderer(monkeypatch):
    import utils
    from model.raster import HardPhongShader, MeshRenderer, SilhouetteRenderer
    net, data, cams, TmpVs, Tmpfs, fids = _scene()
    N, Hh, Ww = fids.numel(), data.H, data.W
    monkeypatch.setitem(sys.modules, "pytorch3d", None)        # any pytorch3d import raises
    with pytest.raises(ImportError):
        import pytorch3d  # noqa: F401
    net.maskRender = _recording(MeshRenderer)(net.maskRender.rasterizer, HardPhongShader(DEV, cams))
    gts = _gts(N, Hh, Ww, image=False)
    colors, imgs, def1imgs, defMeshVs = net.infer(TmpVs, Tmpfs, Hh, Ww, H.RATIO, fids, False, gts)
    V = TmpVs.shape[0]
    assert colors.dtype == np.uint8 and colors.shape == (N, Hh, Ww, 3)
    assert imgs.dtype == np.uint8 and imgs.shape == (N, Hh, Ww, 3)
    assert def1imgs.dtype == np.uint8 and def1imgs.shape == (N, Hh, Ww, 4)
    assert defMeshVs.dtype == np.float32 and defMeshVs.shape == (N, V, 3)
    poses, trans, d_cond, _ = data.get_grad_parameters(fids, DEV)
    with torch.no_grad():
        dv = net.deformer(TmpVs[None].expand(N, -1, 3), [d_cond, [poses, trans]], ratio=H.RATIO)
        d1 = net.deformer.defs[0](TmpVs[None].expand(N, -1, 3), d_cond, ratio=H.RATIO)
    assert np.array_equal(defMeshVs, dv.cpu().numpy())
    c0, c1 = net.maskRender.calls
    assert np.array_equal(c0["verts"].cpu().numpy(), defMeshVs) and c0["cameras"] is None and c0["lights"] is None
    assert torch.equal(c1["verts"], d1)
    tz = float(data.trans.detach().mean(0)[2])
    assert c1["lights"].location.tolist() == [[0., 1., pytest.approx(tz)]]
    front = torch.tensor([[-1., 0., 0.], [0., 1., 0.], [0., 0., -1.]], device=DEV)
    assert torch.equal(c1["cameras"].R, front.expand(N, 3, 3)) and torch.allclose(c1["cameras"].T, data.trans.mean(0).expand(N, 3))
    fc = Tmpfs.cpu().numpy()
    # images: the test's own composition within 1 LSB
    e0 = _composed(c0, fc, _cam_pos(cams, N), [0., 1., 0.], 3)
    e1 = _composed(c1, fc, _cam_pos(c1["cameras"], N), [0., 1., tz], 4)
    d_img = np.abs(imgs.astype(np.int32) - e0).max()
    d_def1 = np.abs(def1imgs.astype(np.int32) - e1).max()
    cov0 = (c0["frags"].pix_to_face[..., 0] >= 0).cpu().numpy()
    cov1 = (c1["frags"].pix_to_face[..., 0] >= 0).cpu().numpy()
    print("infer: %d / %d covered pixels; imgs max %d LSB off, def1imgs max %d LSB off"
          % (cov0.sum(), cov1.sum(), d_img, d_def1))
    assert 500 < cov0.sum() < 0.8 * cov0.size and 500 < cov1.sum() < 0.8 * cov1.size
    assert d_img <= 1 and d_def1 <= 1
    assert np.array_equal(def1imgs[..., 3], np.where(cov1, 255, 0).astype(np.uint8))
    # maskE: IoU of the fragments' coverage with the gt mask
    g = gts['mask'].cpu().numpy().astype(np.float64)
    m = cov0.astype(np.float64)
    iou = 1. - (m * g).reshape(N, -1).sum(1) / (m + g - m * g).reshape(N, -1).sum(1)
    np.testing.assert_allclose(gts['maskE'], iou, rtol=1e-6)
    # colours: infer_rays on FindSurfacePs of the same fragments; 255 elsewhere
    bi, ri, ci, ps, _ = utils.FindSurfacePs(TmpVs, Tmpfs, c0["frags"])
    direct = net.infer_rays(bi, ri, ci, ps, Hh, Ww, H.RATIO, fids).cpu().numpy().astype(np.uint8)
    assert np.array_equal(colors, direct)
    seeded = np.zeros((N, Hh, Ww), bool)
    seeded[bi.cpu().numpy(), ri.cpu().numpy(), ci.cpu().numpy()] = True
    assert seeded.sum() > 500 and np.all(colors[~seeded] == 255) and np.any(colors[seeded] != 255)
    # notcolor: no tracing, same images
    out = net.infer(TmpVs, Tmpfs, Hh, Ww, H.RATIO, fids, True, _gts(N, Hh, Ww, image=False))
    assert out[0] is None and np.array_equal(out[1], imgs) and np.array_equal(out[2], def1imgs)
    # the gt overlay (network.py:327-328, :368-369): BGR into imgs, RGB into colors, outside the rendered mask
    gi = _gts(N, Hh, Ww, image=True)
    col2, img2, _, _ = net.infer(TmpVs, Tmpfs, Hh, Ww, H.RATIO, fids, False, gi)
    im = gi['image'].cpu().numpy()
    bg = ~cov0
    assert np.array_equal(img2[bg], (im[bg][:, [2, 1, 0]] * np.float32(255.)).astype(np.uint8))
    assert np.array_equal(col2[bg], (im[bg] * np.float32(255.)).astype(np.uint8))
    assert np.array_equal(img2[cov0], imgs[cov0]) and np.array_equal(col2[cov0], colors[cov0])
    # the default SilhouetteRenderer: images are its silhouettes, colours unchanged
    net.maskRender = SilhouetteRenderer(net.maskRender.rasterizer)
    col3, img3, def3, vs3 = net.infer(TmpVs, Tmpfs, Hh, Ww, H.RATIO, fids, False, _gts(N, Hh, Ww, image=False))
    assert np.array_equal(img3, np.repeat(np.where(cov0, 255, 0).astype(np.uint8)[..., None], 3, -1))
    assert np.array_equal(def3, np.repeat(np.where(cov1, 255, 0).astype(np.uint8)[..., None], 4, -1))
    assert np.array_equal(col3, colors) and np.array_equal(vs3, defMeshVs)
