"""CPU: the float64 restatement of pytorch3d's vertex normals and HardPhongShader (tests/mesh_shade_ref.py) against
hand-derived closed forms, the pytorch3d defaults of the built-in renderer classes, and the C layout of
sr_phong_params."""
import ctypes
import math
import os
import subprocess
import tempfile

import numpy as np

import helpers
from mesh_shade_ref import shade_phong_p3d, vertex_normals_p3d

# one triangle in the z = 0 plane; (v2-v1) x (v0-v1) = (0, 0, 4): it faces +z
TRI_V = np.array([[-1., -1., 0.], [1., -1., 0.], [0., 1., 0.]])
TRI_F = np.array([[0, 1, 2]])
THIRD = np.full(3, 1. / 3.)
P = TRI_V.mean(0)                       # the pixel's surface point (barycentrics 1/3)


def _shade(light, cam, colors=None, **kw):
    vs = TRI_V[None]
    img, terms = shade_phong_p3d(vs, vertex_normals_p3d(vs, TRI_F), TRI_F, np.zeros((1, 1, 1), np.int64),
                                 THIRD.reshape(1, 1, 1, 3), np.array([cam]), np.array([light]), colors=colors, **kw)
    return img[0, 0, 0], {k: v[0, 0, 0] for k, v in terms.items()}


def _dir(angle):
    return np.array([math.sin(angle), 0., math.cos(angle)])


def test_single_triangle_closed_forms():
    th, psi = math.radians(35.), math.radians(25.)
    light = P + 2.0 * _dir(th)                 # light at angle theta from the normal, in the x-z plane
    cam = P + 3.0 * _dir(-psi)                 # eye on the other side of the normal
    rgb, t = _shade(light, cam)
    # reflected ray r = (-sin theta, 0, cos theta), view v = (-sin psi, 0, cos psi): cos phi = v.r = cos(theta - psi)
    phi = th - psi
    assert abs(t["cos"] - math.cos(th)) < 1e-12
    np.testing.assert_allclose(t["diffuse"], 0.3 * math.cos(th), rtol=0, atol=1e-12)
    np.testing.assert_allclose(t["specular"], 0.2 * math.cos(phi) ** 64, rtol=1e-10, atol=0)
    np.testing.assert_allclose(rgb[:3], 0.5 + 0.3 * math.cos(th) + 0.2 * math.cos(phi) ** 64, rtol=1e-12)
    assert rgb[3] == 1.0


def test_mirror_direction_gives_full_highlight():
    th = math.radians(20.)
    rgb, t = _shade(P + 1.5 * _dir(th), P + 4.0 * _dir(-th))   # the eye sits on the reflected ray: cos phi = 1
    np.testing.assert_allclose(t["specular"], 0.2, rtol=1e-12)
    np.testing.assert_allclose(rgb[:3], 0.5 + 0.3 * math.cos(th) + 0.2, rtol=1e-12)


def test_light_behind_face_gives_ambient_only():
    tex = np.array([0.2, 0.6, 0.9])
    cols = np.tile(tex, (1, 3, 1))
    rgb, t = _shade(P - 2.0 * _dir(math.radians(10.)), P + 3.0 * _dir(0.), colors=cols)
    assert t["cos"] < 0
    assert np.all(t["specular"] == 0) and np.all(t["diffuse"] == 0)
    np.testing.assert_allclose(rgb[:3], 0.5 * tex, rtol=1e-15)   # up to the barycentric sum of the texel


def test_texel_scales_ambient_and_diffuse_not_specular():
    th = math.radians(20.)
    tex = np.array([0.25, 0.5, 1.0])
    rgb, t = _shade(P + 1.5 * _dir(th), P + 4.0 * _dir(-th), colors=np.tile(tex, (1, 3, 1)))
    np.testing.assert_allclose(rgb[:3], (0.5 + 0.3 * math.cos(th)) * tex + 0.2, rtol=1e-12)


def test_background_pixels():
    vs = TRI_V[None]
    img, _ = shade_phong_p3d(vs, vertex_normals_p3d(vs, TRI_F), TRI_F, -np.ones((1, 2, 3), np.int64),
                             -np.ones((1, 2, 3, 3)), np.zeros((1, 3)), np.zeros((1, 3)))
    assert np.array_equal(img, np.tile([1., 1., 1., 0.], (1, 2, 3, 1)))


def test_vertex_normals_area_weighted_and_unreferenced_zero():
    # two faces sharing the edge (0,1): a large one in z = 0 (normal +z) and a small one in x = 0 (normal +x)
    vs = np.array([[0., 0., 0.], [0., 1., 0.], [-3., 0., 0.], [0., 0., 0.5], [7., 7., 7.]])
    fs = np.array([[0, 1, 2], [0, 1, 3]])
    a = np.cross(vs[2] - vs[1], vs[0] - vs[1])
    b = np.cross(vs[3] - vs[1], vs[0] - vs[1])
    np.testing.assert_allclose(a, [0, 0, 3])         # twice the area 1.5
    np.testing.assert_allclose(b, [0.5, 0, 0])       # twice the area 0.25
    n = vertex_normals_p3d(vs, fs)
    np.testing.assert_allclose(n[0], (a + b) / np.linalg.norm(a + b), rtol=1e-14)
    np.testing.assert_allclose(n[2], [0, 0, 1])
    np.testing.assert_allclose(n[3], [1, 0, 0])
    assert np.array_equal(n[4], np.zeros(3))          # unreferenced vertex
    nu = vertex_normals_p3d(vs, fs, unit_faces=True)  # the unit-face rule gives the bisector instead
    np.testing.assert_allclose(nu[0], np.array([1., 0., 1.]) / math.sqrt(2.), rtol=1e-14)
    # a zero-area face (repeated index) adds nothing
    n2 = vertex_normals_p3d(vs, np.concatenate([fs, [[0, 0, 1]]]))
    np.testing.assert_allclose(n2, n, rtol=0, atol=0)


def test_renderer_defaults_match_pytorch3d():
    helpers.dropin()
    from model.raster import BlendParams, HardPhongShader, Materials, PointLights
    lt, mt, bp = PointLights(), Materials(), BlendParams()
    assert lt.location.tolist() == [[0., 1., 0.]]
    assert (lt.ambient_color, lt.diffuse_color, lt.specular_color) == ((0.5,) * 3, (0.3,) * 3, (0.2,) * 3)
    assert (mt.ambient_color, mt.diffuse_color, mt.specular_color, mt.shininess) == ((1.,) * 3, (1.,) * 3, (1.,) * 3, 64.)
    assert bp.background_color == (1., 1., 1.) and (bp.sigma, bp.gamma) == (1e-4, 1e-4)
    sh = HardPhongShader()
    assert sh.cameras is None
    assert sh.lights.location.tolist() == [[0., 1., 0.]] and sh.materials.shininess == 64.
    assert sh.blend_params.background_color == (1., 1., 1.)
    p = sh.params(sh.lights, sh.materials, sh.blend_params)
    got = [list(getattr(p, k)) for k in ("light_ambient", "light_diffuse", "light_specular", "mat_ambient",
                                         "mat_diffuse", "mat_specular", "background")]
    np.testing.assert_allclose(got, [[0.5] * 3, [0.3] * 3, [0.2] * 3, [1.] * 3, [1.] * 3, [1.] * 3, [1.] * 3],
                               rtol=1e-7)
    assert p.shininess == 64.
    # pytorch3d keyword names, per-frame locations
    lt2 = PointLights(device="cpu", location=((0, 1, 2.5), (1, 0, 0)), ambient_color=((0.1, 0.2, 0.3),))
    assert lt2.location.shape == (2, 3) and lt2.ambient_color == (0.1, 0.2, 0.3)


def test_phong_params_layout_matches_c():
    from selfreconcode_b200 import _lib
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "selfrecon_b200.h"\nint main(){printf("%zu %zu %zu\\n",' \
          'sizeof(sr_phong_params),offsetof(sr_phong_params,shininess),offsetof(sr_phong_params,background));}'
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(helpers.ROOT, "include"), c, "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(_lib.PhongParams), _lib.PhongParams.shininess.offset,
                     _lib.PhongParams.background.offset]
