"""CPU: the float64 rasteriser restatement (tests/raster_ref.py) against closed forms: lattice-point counts under the
inclusive rule, perspective-correct barycentrics and depth, the tie rule, winding independence, and its own
watertightness on the crack scene of test_gpu_raster_contract."""
import math

import numpy as np
import pytest

import raster_ref as ref


def _one(verts, faces, H, W):
    r = ref.raster(np.asarray(verts, np.float32)[None], faces, H, W)
    return r.face[0], r


@pytest.mark.parametrize("k", [1, 2, 5, 16])
def test_half_square_counts(k):
    """A k x k square with integer corners split along its diagonal: the closed lower half holds (k+1)(k+2)/2 pixel
    centres, the upper half the rest of the (k+1)^2 (the diagonal goes to the lower id, both lie at depth 1)."""
    o = 3
    v = [(o, o, 1.), (o + k, o, 1.), (o + k, o + k, 1.), (o, o + k, 1.)]
    for a, b in (((0, 1, 2), (0, 2, 3)), ((0, 2, 3), (0, 1, 2))):
        face, r = _one(v, [a, b], 24, 24)
        half = (k + 1) * (k + 2) // 2
        assert (face == 0).sum() == half and (face == 1).sum() == half - (k + 1)
        assert (face >= 0).sum() == (k + 1) ** 2
        # integer vertices: every edge value is exact in fp32, so only the diagonal, where both faces lie at depth 1
        # and their fp32 depths may differ in the last bit, is sensitive
        diag = np.zeros((24, 24), bool)
        diag[np.arange(o, o + k + 1), np.arange(o, o + k + 1)] = True
        assert np.array_equal(r.sensitive[0], diag)
    face, _ = _one(v, [(0, 1, 2)], 24, 24)
    assert (face == 0).sum() == (k + 1) * (k + 2) // 2


def test_lattice_triangles_pick():
    """Random integer triangles: the closed triangle holds A + B/2 + 1 lattice points (Pick), B = sum gcd(|dx|, |dy|)."""
    rng = np.random.default_rng(1)
    for _ in range(40):
        p = rng.integers(0, 30, (3, 2)).astype(np.float64)
        A2 = (p[1, 0] - p[0, 0]) * (p[2, 1] - p[0, 1]) - (p[2, 0] - p[0, 0]) * (p[1, 1] - p[0, 1])
        if A2 == 0:
            continue
        B = sum(math.gcd(int(abs(p[i, 0] - p[(i + 1) % 3, 0])), int(abs(p[i, 1] - p[(i + 1) % 3, 1]))) for i in range(3))
        want = abs(A2) / 2 + B / 2 + 1
        v = np.concatenate([p, np.full((3, 1), 2.)], 1)
        face, r = _one(v, [(0, 1, 2)], 32, 32)
        assert (face == 0).sum() == want
        face2, _ = _one(v, [(0, 2, 1)], 32, 32)           # winding does not matter
        assert np.array_equal(face, face2)
        assert not r.sensitive.any()


def test_representable_edges():
    """Right triangle (0,0), (8,0), (0,4) at offset 2: x + 2y <= 8 holds 25 lattice points; a half-pixel triangle holds
    exactly its vertex-free interior points."""
    face, _ = _one([(2, 2, 1.), (10, 2, 1.), (2, 6, 1.)], [(0, 1, 2)], 16, 16)
    assert (face == 0).sum() == 25
    face, _ = _one([(0.5, 0.5, 1.), (6.5, 0.5, 1.), (0.5, 6.5, 1.)], [(0, 1, 2)], 16, 16)
    # x, y >= 1 and x + y <= 7 - 0.5 + 0.5 = 7: points (x, y) with x, y in [1, 6], x + y <= 7 -> 21
    assert (face == 0).sum() == 21


def test_perspective_barycentrics_and_depth():
    """b_i = (l_i / z_i) / sum(l_j / z_j), z = 1 / sum(l_j / z_j), with l the screen barycentrics from a 2x2 solve;
    the interpolated camera-space point (b-weighted) projects back onto the pixel."""
    v = np.array([(2.25, 3.5, 1.5), (40.75, 9.0, 4.0), (12.5, 37.25, 9.0)])
    face, r = _one(v, [(0, 1, 2)], 48, 48)
    rr, cc = np.nonzero(face == 0)
    assert len(rr) > 400
    M = np.array([[v[0, 0] - v[2, 0], v[1, 0] - v[2, 0]], [v[0, 1] - v[2, 1], v[1, 1] - v[2, 1]]])
    l01 = np.linalg.solve(M, np.stack([cc - v[2, 0], rr - v[2, 1]]))
    l = np.stack([l01[0], l01[1], 1 - l01[0] - l01[1]], 1)
    q = l / v[:, 2]
    want_b = q / q.sum(1, keepdims=True)
    want_z = 1 / q.sum(1)
    assert np.abs(r.bary[0][rr, cc] - want_b).max() < 1e-12
    assert np.abs(r.zbuf[0][rr, cc] - want_z).max() < 1e-12
    # perspective: with x = X f / Z, the camera-space point sum b_i (x_i z_i, y_i z_i, z_i) projects to the pixel
    Pc = (want_b[:, :, None] * np.stack([v[:, 0] * v[:, 2], v[:, 1] * v[:, 2], v[:, 2]], 1)[None]).sum(1)
    assert np.abs(Pc[:, 0] / Pc[:, 2] - cc).max() < 1e-9 and np.abs(Pc[:, 1] / Pc[:, 2] - rr).max() < 1e-9
    assert (r.bary_bound[0][rr, cc] > 0).all() and (r.z_bound[0][rr, cc] < 1e-5 * want_z).all()


def test_tie_rule_and_winding():
    tri = [(2, 2, 2.), (20, 3, 2.), (5, 18, 2.)]
    v = tri + [(x, y, z - 1) for x, y, z in tri]
    # nearer face wins whatever its id
    face, _ = _one(v, [(0, 1, 2), (3, 4, 5)], 24, 24)
    assert set(np.unique(face)) == {-1, 1}
    face, _ = _one(v, [(3, 4, 5), (0, 1, 2)], 24, 24)
    assert set(np.unique(face)) == {-1, 0}
    # exact tie: the lower id, for either order of the duplicate; a reversed duplicate covers the same pixels
    for fs in ([(0, 1, 2), (0, 1, 2)], [(0, 1, 2), (0, 2, 1)], [(0, 2, 1), (0, 1, 2)]):
        face, r = _one(tri, fs, 24, 24)
        assert set(np.unique(face)) == {-1, 0}
    f1, r1 = _one(tri, [(0, 1, 2)], 24, 24)
    f2, r2 = _one(tri, [(0, 2, 1)], 24, 24)
    assert np.array_equal(f1, f2)
    assert np.allclose(r1.bary[0][f1 >= 0][:, [0, 2, 1]], r2.bary[0][f2 >= 0], rtol=0, atol=1e-15)
    # frames: ids n F + f
    vs = np.stack([np.asarray(tri, np.float32), np.asarray(tri, np.float32) + [1, 0, 0]])
    r = ref.raster(vs, [(0, 1, 2)], 24, 24)
    assert set(np.unique(r.face[1])) == {-1, 1}


def test_dropped_faces():
    for z in (0., 1e-8, -1., np.nan, np.inf):
        face, _ = _one([(2, 2, 1.), (20, 3, 1.), (5, 18, z)], [(0, 1, 2)], 24, 24)
        assert (face < 0).all(), z
    face, _ = _one([(2, 2, 1.), (20, 3, 1.), (11, 2.5, 1.)], [(0, 1, 2), (0, 1, 1)], 24, 24)   # collinear, repeated
    assert (face < 0).all()
    r = ref.raster(np.zeros((0, 3, 3), np.float32), [(0, 1, 2)], 4, 5)
    assert r.face.shape == (0, 4, 5)
    r = ref.raster(np.zeros((2, 3, 3), np.float32), np.zeros((0, 3), np.int64), 4, 5)
    assert (r.face == -1).all() and (r.zbuf == -1).all()


def test_crack_scene_watertight():
    """In float64 the two faces of every quad cover every pixel centre inside the quad (closed), the diagonal's centres
    are must-cover, and the bounds mark them sensitive unless the diagonal is exact in fp32."""
    verts, faces, side = ref.crack_scene(grid=24, n_frames=2, seed=5)
    r = ref.raster(verts, faces, side, side)
    F = faces.shape[0]
    for n in range(2):
        v = verts[n].astype(np.float64)
        A, B, C, D = (v[k::4] for k in range(4))
        yy, xx = np.mgrid[0:side, 0:side].astype(np.float64)
        cell = (yy // 7) * 24 + xx // 7
        q = cell.astype(np.int64)

        def e(a, b):
            return (a[q, 0] - xx) * (b[q, 1] - yy) - (b[q, 0] - xx) * (a[q, 1] - yy)
        s = np.sign(e(A, C))
        inside = (s * e(A, C) >= 0) & (s * e(C, B) >= 0) & (s * e(B, D) >= 0) & (s * e(D, A) >= 0)
        face = r.face[n]
        assert (face[inside] >= 0).all() and (face[~inside] < 0).all()
        assert ((face[inside] - n * F) // 2 == q[inside]).all()
        # centres exactly on a diagonal (the quads whose endpoints are fp32 numbers): covered by both faces, must-cover
        on_exact = (e(A, B) == 0) & inside
        assert on_exact.sum() > 24 and r.must_cover[n][on_exact].all()
        assert (face[on_exact] % 2 == 0).all()           # both at the same depth there: the lower id
        # must-cover centres lie within rounding of a diagonal, inside their quad
        mc = r.must_cover[n]
        assert not mc[~inside].any() and (np.abs(e(A, B))[mc] < 1e-4).all()
        assert (mc & ~on_exact).sum() > 0
    assert (r.sensitive & r.must_cover).sum() > 0
