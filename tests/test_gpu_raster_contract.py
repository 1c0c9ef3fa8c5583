"""GPU: the mesh rasteriser (csrc/raster.cu, ops.raster_mesh) against the float64 restatement (tests/raster_ref.py) and,
bit for bit, against its fp32 twin oracle.raster_mesh.  Bars on every scene: the float64 face choice on every pixel that
is not sensitive; no must-cover pixel left empty; every covered pixel with barycentrics >= 0 summing to 1 within 4 ulp
and a positive depth; barycentrics and depth within the formula's fp32 rounding bound.  Then invariances (winding,
vertex rotation, face order, duplicate faces, frame batching, rerun) and negative controls, each of which must fail
its bar."""
import ctypes as C

import numpy as np
import pytest
import torch

import helpers as H
import raster_ref as ref
import texture_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
ULP1 = 2.0 ** -23


def kernel(vs, faces, Hh, Ww):
    """sr_raster_mesh on outputs pre-filled with sentinels (ids -7, NaN barycentrics and depth, a garbage key image)
    -> numpy (face [N,H,W] int64, bary [N,H,W,3] float32, zbuf [N,H,W] float32)."""
    from selfreconcode_b200 import _lib
    vs = torch.as_tensor(np.asarray(vs, np.float32), device=DEV).contiguous()
    fc = torch.as_tensor(np.asarray(faces, np.int64).reshape(-1, 3), device=DEV).contiguous()
    N, V, F = vs.shape[0], vs.shape[1], fc.shape[0]
    keys = torch.full((N, Hh, Ww), 12345, dtype=torch.int64, device=DEV)
    p2f = torch.full((N, Hh, Ww), -7, dtype=torch.int64, device=DEV)
    bary = torch.full((N, Hh, Ww, 3), float("nan"), device=DEV)
    zbuf = torch.full((N, Hh, Ww), float("nan"), device=DEV)
    p = lambda t: C.c_void_p(t.data_ptr())            # noqa: E731
    rc = _lib.load().sr_raster_mesh(p(vs), p(fc), N, V, F, Hh, Ww, p(keys), p(p2f), p(bary), p(zbuf),
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    return p2f.cpu().numpy(), bary.cpu().numpy(), zbuf.cpu().numpy()


def bars(name, got, r, vs=None, faces=None, oracle=True):
    """The contract's bars on one scene; returns the largest error / bound ratio."""
    face, bary, zbuf = got
    ns = ~r.sensitive
    cov = face >= 0
    differ = int(((face != r.face) & ns).sum())
    holes = int((r.must_cover & ~cov).sum())
    bsum = np.abs(bary.astype(np.float64).sum(-1) - 1.)[cov]
    ok = cov & ns & (face == r.face)
    with np.errstate(divide="ignore", invalid="ignore"):
        rb = np.abs(bary.astype(np.float64) - r.bary)[ok] / r.bary_bound[ok]
        rz = np.abs(zbuf.astype(np.float64) - r.zbuf)[ok] / r.z_bound[ok]
    rb, rz = np.nan_to_num(rb, posinf=np.inf), np.nan_to_num(rz, posinf=np.inf)
    ratio = float(max(rb.max(initial=0.), rz.max(initial=0.)))
    print("%s: %d pixels, %d covered, %d sensitive, %d must-cover, %d outline; %d differ off the sensitive set, %d "
          "must-cover left empty; max |sum b - 1| %.1f ulp; max error / bound %.3f"
          % (name, face.size, cov.sum(), r.sensitive.sum(), r.must_cover.sum(), r.outline.sum(), differ, holes,
             bsum.max(initial=0.) / ULP1, ratio))
    assert differ == 0 and holes == 0
    assert (bary[cov] >= 0).all() and (bsum <= 4 * ULP1).all() and (zbuf[cov] > 0).all()
    assert (bary[~cov] == -1).all() and (zbuf[~cov] == -1).all() and (face >= -1).all()
    assert ratio <= 1.
    if oracle:
        from oracle import oracle as O
        F = np.asarray(faces).reshape(-1, 3).shape[0]
        for n in range(face.shape[0]):
            po, bo, zo = O.raster_mesh(np.asarray(vs[n], np.float32), faces, face.shape[1], face.shape[2])
            fn = np.where(face[n] >= 0, face[n] - n * F, -1)
            assert np.array_equal(fn, po), (name, n, int((fn != po).sum()))
            assert np.array_equal(bary[n].view(np.uint32), bo.view(np.uint32)), (name, n)
            assert np.array_equal(zbuf[n].view(np.uint32), zo.view(np.uint32)), (name, n)
    return ratio


def run(name, vs, faces, Hh, Ww, oracle=True):
    vs = np.asarray(vs, np.float32)
    r = ref.raster(vs, faces, Hh, Ww)
    got = kernel(vs, faces, Hh, Ww)
    bars(name, got, r, vs, faces, oracle)
    return got, r


# ---- (a) crack scene --------------------------------------------------------------------------------------------------
def test_crack_scene():
    """22,500 disjoint quads per frame, each split along a diagonal through pixel centres (raster_ref.crack_scene),
    N = 3: no centre on a shared diagonal may be left empty; then frame batching and rerun are bitwise."""
    vs, faces, side = ref.crack_scene(150, 3, seed=11)
    assert faces.shape[0] // 2 >= 20000
    got, r = run("crack scene", vs, faces, side, side)
    assert r.must_cover.sum() > 10000
    again = kernel(vs, faces, side, side)
    for a, b in zip(got, again):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    F = faces.shape[0]
    for n in range(3):
        one = kernel(vs[n:n + 1], faces, side, side)
        assert np.array_equal(np.where(got[0][n] >= 0, got[0][n] - n * F, -1), one[0][0])
        assert np.array_equal(got[1][n].view(np.uint32), one[1][0].view(np.uint32))
        assert np.array_equal(got[2][n].view(np.uint32), one[2][0].view(np.uint32))


def test_crack_scene_negative_controls():
    """The strict (> 0) rule and the contracted edge function each leave must-cover centres empty."""
    vs, faces, side = ref.crack_scene(60, 2, seed=12)
    r = ref.raster(vs, faces, side, side)
    for kw in (dict(strict=True), dict(contract=True)):
        face = ref.fp32_raster(vs, faces, side, side, **kw)[0]
        holes = int((r.must_cover & (face < 0)).sum())
        print("negative control %s: %d of %d must-cover centres empty" % (kw, holes, r.must_cover.sum()))
        assert holes > 0
    face = ref.fp32_raster(vs, faces, side, side)[0]
    assert not (r.must_cover & (face < 0)).any()


# ---- (b) closed template ----------------------------------------------------------------------------------------------
_TPL = {}


def template(Hh, Ww):
    if (Hh, Ww) not in _TPL:
        from test_gpu_mesh_shade import _scene
        from test_gpu_texture import deformed
        H.dropin()
        from model.raster import screen_vertices
        net, data, cams, TmpVs, Tmpfs, _ = _scene(Hh, Ww, 3)
        with torch.no_grad():
            data.poses[:, 0, 1] = torch.linspace(-0.6, 0.6, 3, device=DEV)
        D = deformed(net, data, TmpVs, [0, 1, 2])
        with torch.no_grad():
            s = screen_vertices(D, cams)
        _TPL[(Hh, Ww)] = (s.float().cpu().numpy(), Tmpfs.long().cpu().numpy())
    return _TPL[(Hh, Ww)]


@pytest.mark.parametrize("Hh,Ww", [(512, 512), (112, 96)])
def test_template(Hh, Ww):
    from selfreconcode_b200 import ops
    vs, faces = template(Hh, Ww)
    got, r = run("template %dx%d" % (Hh, Ww), vs, faces, Hh, Ww)
    assert (got[0] >= 0).sum() > 0.05 * got[0].size
    p2f, bary, zbuf = ops.raster_mesh(torch.from_numpy(vs).to(DEV), torch.from_numpy(faces).to(DEV), Hh, Ww)
    assert np.array_equal(p2f[..., 0].cpu().numpy(), got[0])
    assert np.array_equal(bary[..., 0, :].cpu().numpy().view(np.uint32), got[1].view(np.uint32))
    assert np.array_equal(zbuf[..., 0].cpu().numpy().view(np.uint32), got[2].view(np.uint32))


def test_template_invariances():
    """On the 112 x 96 template: reversed winding and rotated vertex order keep the coverage bitwise, and barycentrics /
    depth within the rounding of the reordered sum (and, rotated, of the area's other formula); a face permutation changes ids only through it (and at exact depth-bit ties); a higher-id
    duplicate of every face never wins."""
    Hh, Ww = 112, 96
    vs, faces = template(Hh, Ww)
    F = faces.shape[0]
    base = kernel(vs, faces, Hh, Ww)
    r = ref.raster(vs, faces, Hh, Ww)
    cov = base[0] >= 0

    fid = np.where(cov, base[0] - np.arange(3)[:, None, None] * F, 0)
    Tv = vs.astype(np.float64)[np.arange(3)[:, None, None, None], faces[fid]]          # [3,H,W,3 vertices,3]
    (x0, y0), (x1, y1), (x2, y2) = [(Tv[..., k, 0], Tv[..., k, 1]) for k in range(3)]
    A, eA = ref.edge(x1, y1, x2, y2, x0, y0)
    for perm_v, name in (([0, 2, 1], "reversed"), ([1, 2, 0], "rotated")):
        got = kernel(vs, faces[:, perm_v], Hh, Ww)
        assert np.array_equal(got[0] >= 0, cov), name
        same = (got[0] == base[0]) & cov
        assert not ((got[0] != base[0]) & ~r.sensitive).any()
        back = np.empty_like(got[1])
        back[..., perm_v] = got[1]
        # the edge values are the same bits; the area is the exact negation when reversed, and another formula (with
        # its own rounding e_A') when rotated, which scales every l_i, hence the depth, by 1 + O((e_A + e_A') / |A|)
        # and leaves b = q / sum(q) unscaled.  s = q0 + q1 + q2 changes its order: each order rounds s twice (within
        # 2u s, all q_i >= 0), so 1 / s moves by at most 4u / s, and each division adds half an ulp.
        dA = 0. if name == "reversed" else (eA + ref.edge(x2, y2, x0, y0, x1, y1)[1]) / np.abs(A)
        b0, z0 = base[1][same].astype(np.float64), base[2][same].astype(np.float64)
        bb = 4 * ref.U * b0 + np.spacing(base[1][same])
        bz = (4 * ref.U + (dA[same] if name == "rotated" else 0.)) * z0 + np.spacing(base[2][same])
        eb = (np.abs(back[same] - b0) / bb).max()
        ez = (np.abs(got[2][same] - z0) / bz).max()
        print("%s vertex order: max error / bound %.2f (barycentrics), %.2f (depth); %.1f / %.1f ulp"
              % (name, eb, ez, (np.abs(back[same] - b0) / np.spacing(base[1][same])).max(),
                 (np.abs(got[2][same] - z0) / np.spacing(base[2][same])).max()))
        assert eb <= 1 and ez <= 1, name
    rng = np.random.default_rng(3)
    perm = rng.permutation(F)
    got = kernel(vs, faces[perm], Hh, Ww)
    frame = np.arange(3)[:, None, None] * F
    mapped = np.where(got[0] >= 0, perm[np.maximum(got[0] - frame, 0)] + frame, -1)
    assert np.array_equal(got[2].view(np.uint32), base[2].view(np.uint32))
    low = ref.fp32_raster(vs, faces, Hh, Ww)[0]
    high = ref.fp32_raster(vs, faces, Hh, Ww, ties_to_last=True)[0]
    ties = low != high
    assert not ((mapped != base[0]) & ~ties).any()
    print("face permutation: %d pixels differ, %d exact depth-bit ties" % ((mapped != base[0]).sum(), ties.sum()))
    dup = kernel(vs, np.concatenate([faces, faces]), Hh, Ww)
    assert np.array_equal(np.where(dup[0] >= 0, dup[0] - 2 * frame, -1), np.where(cov, base[0] - frame, -1))
    assert np.array_equal(dup[1].view(np.uint32), base[1].view(np.uint32))


def test_template_negative_controls():
    """Screen-space barycentrics fail the barycentric bound; swapped row and column fail the face choice on 112 x 96."""
    Hh, Ww = 112, 96
    vs, faces = template(Hh, Ww)
    r = ref.raster(vs, faces, Hh, Ww)
    face, bary, _ = ref.fp32_raster(vs, faces, Hh, Ww, screen_bary=True)
    ok = (face == r.face) & (face >= 0) & ~r.sensitive
    ratio = (np.abs(bary.astype(np.float64) - r.bary)[ok] / r.bary_bound[ok]).max()
    print("negative control, screen-space barycentrics: max error / bound %.3g" % ratio)
    assert ratio > 100
    face = ref.fp32_raster(vs[..., [1, 0, 2]], faces, Hh, Ww)[0]
    differ = int(((face != r.face) & ~r.sensitive).sum())
    print("negative control, swapped row and column: %d pixels differ" % differ)
    assert differ > 1000


# ---- (c) UV layouts ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,R", [("chart", 1024), ("seam", 512)])
def test_uv_layouts(name, R):
    from test_gpu_texture import layout, scene
    _, _, _, TmpVs, Tmpfs = scene(96, 2)
    vt, ft = layout(name, TmpVs, Tmpfs)
    xy = texture_ref.uv_screen(vt, R)           # the baker's fp32 atlas vertices (u R - 0.5, (1 - v) R - 0.5)
    vs = np.concatenate([xy, np.ones((xy.shape[0], 1))], 1)[None]
    run("UV %s R=%d" % (name, R), vs, ft, R, R)


# ---- (d) edge cases ---------------------------------------------------------------------------------------------------
def _edge_scenes():
    tri = [(2.3, 1.7, 2.), (17.6, 4.2, 3.), (6.1, 13.9, 1.5)]
    out = {}
    for z in (0., 1e-8, -1.):
        out["vertex at z = %g" % z] = ([tri[0], tri[1], (6.1, 13.9, z)] + tri, [(0, 1, 2), (3, 4, 5)], 16, 20)
    out["vertex at z = 2e-8"] = ([tri[0], tri[1], (6.1, 13.9, 2e-8)], [(0, 1, 2)], 16, 20)
    big = [(-1e9, -1e9, 2.), (1e9, 3., 2.), (5., 1e9, 2.), (-3e8, 7., 1.), (12., -2e8, 1.5), (2e8, 2e8, 3.),
           (-50., 5., 1.), (-20., 30., 1.), (-40., -9., 1.)]
    out["faces up to 1e9 and off screen"] = (big, [(0, 1, 2), (3, 4, 5), (6, 7, 8)], 24, 31)
    out["degenerate, collinear, repeated index"] = (
        tri + [(1., 1., 1.), (9., 5., 1.), (17., 9., 1.), (3.3, 2.2, 1.), (3.3, 2.2, 1.)],
        [(3, 4, 5), (0, 0, 1), (6, 7, 2), (6, 6, 6), (0, 1, 2), (1, 1, 2)], 16, 20)
    out["coincident duplicates"] = (tri, [(0, 1, 2), (0, 1, 2), (1, 2, 0), (0, 2, 1)], 16, 20)
    out["centres on representable vertices and edges"] = (
        [(2., 2., 1.), (10., 2., 2.), (2., 10., 3.), (10., 10., 1.), (6., 6., 1.5), (14., 2., 1.)],
        [(0, 1, 2), (1, 3, 2), (1, 5, 3), (0, 1, 4)], 14, 16)
    out["H = 1"] = ([(-1., -0.5, 1.), (9., 0., 1.), (0., 0.5, 1.), (3., -2., 2.), (5., 0., 2.), (4., 3., 2.)],
                    [(0, 1, 2), (3, 4, 5)], 1, 12)
    out["W = 1"] = ([(-0.5, -1., 1.), (0., 9., 1.), (0.5, 0., 1.)], [(0, 1, 2)], 12, 1)
    out["H = W = 1"] = ([(-1., -1., 1.), (2., 0., 1.), (0., 2., 1.)], [(0, 1, 2)], 1, 1)
    return out


@pytest.mark.parametrize("name", list(_edge_scenes()))
def test_edge_cases(name):
    v, f, Hh, Ww = _edge_scenes()[name]
    vs = np.asarray(v, np.float32)[None].repeat(2, 0)
    vs[1, :, :2] += np.float32(0.25)
    run(name, vs, f, Hh, Ww)


def test_non_finite_vertex():
    """A face with a NaN or inf vertex covers nothing and leaves the others' result bit for bit unchanged."""
    tri = [(2.3, 1.7, 2.), (17.6, 4.2, 3.), (6.1, 13.9, 1.5), (3., 3., 1.), (12., 6., 1.)]
    base = kernel(np.asarray(tri, np.float32)[None], [(0, 1, 2)], 16, 20)
    assert (base[0] >= 0).sum() > 50
    for bad in (np.nan, np.inf, -np.inf):
        for k in range(3):
            v = np.asarray(tri + [(8., 8., 1.)], np.float32)
            v[5, k] = bad
            got, r = run("vertex %s in coordinate %d" % (bad, k), v[None], [(3, 4, 5), (0, 1, 2), (5, 4, 3)], 16, 20)
            assert np.array_equal(np.where(got[0] >= 0, got[0] - 1, -1), base[0])
            assert np.array_equal(got[1].view(np.uint32), base[1].view(np.uint32))


def test_duplicate_face_tie_control():
    """A coincident duplicate with a higher id never wins; with ties going to the highest id (the negative control)
    it wins every pixel."""
    v, f, Hh, Ww = _edge_scenes()["coincident duplicates"]
    vs = np.asarray(v, np.float32)[None]
    got = kernel(vs, [(0, 1, 2), (0, 1, 2)], Hh, Ww)
    cov = got[0] >= 0
    assert cov.sum() > 50 and (got[0][cov] == 0).all()
    bad = ref.fp32_raster(vs, [(0, 1, 2), (0, 1, 2)], Hh, Ww, ties_to_last=True)[0]
    print("negative control, ties to the highest id: %d of %d pixels go to the duplicate" % ((bad == 1).sum(), cov.sum()))
    assert (bad[cov] == 1).all()


def test_empty_inputs():
    from selfreconcode_b200 import ops
    vs = torch.rand(2, 5, 3, device=DEV)
    p2f, bary, zbuf = ops.raster_mesh(vs, torch.zeros((0, 3), dtype=torch.int64, device=DEV), 7, 9)
    assert p2f.shape == (2, 7, 9, 1) and (p2f == -1).all() and (bary == -1).all() and (zbuf == -1).all()
    assert bary.shape == (2, 7, 9, 1, 3) and zbuf.shape == (2, 7, 9, 1)
    p2f, bary, zbuf = ops.raster_mesh(torch.zeros((0, 5, 3), device=DEV), torch.tensor([[0, 1, 2]], device=DEV), 7, 9)
    assert p2f.shape == (0, 7, 9, 1) and bary.shape == (0, 7, 9, 1, 3) and zbuf.shape == (0, 7, 9, 1)
