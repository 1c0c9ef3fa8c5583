"""CPU: the float64 restatement of the soft point silhouette (tests/points_silhouette_ref.py) against closed forms, and
the hierarchy switch installing the built-in point renderer with pytorch3d unimportable."""
import sys

import numpy as np
import pytest
import torch

import helpers as H
import points_silhouette_ref as ref


def scr(pts, Hh, Ww):
    """(col, row, Z) rows of one frame -> [1,V,3] NDC."""
    return ref.screen_to_ndc(np.asarray(pts, np.float64)[None], Hh, Ww)


def test_projection_matches_screen_convention():
    """K-matrix NDC of a camera equals the built-in (col, row) projection mapped through PixToNdc."""
    g = np.random.default_rng(0)
    Hh, Ww = 40, 56
    v = g.normal(size=(1, 50, 3)) * 0.3
    R = np.diag([-1., -1., 1.])[None]
    T = np.array([[0.1, -0.05, 2.5]])
    focal, pp = np.array([[60., 58.]]), np.array([[27.5, 21.0]])
    ndc = ref.project_ndc(v, R, T, focal, pp, Hh, Ww)
    view = v[0] @ R[0] + T[0]
    col = pp[0, 0] - focal[0, 0] * view[:, 0] / view[:, 2]
    row = pp[0, 1] - focal[0, 1] * view[:, 1] / view[:, 2]
    np.testing.assert_allclose(ndc, scr(np.stack([col, row, view[:, 2]], 1), Hh, Ww), atol=1e-12)


def test_one_point_on_a_pixel_centre():
    Hh = Ww = 9
    r = 2.5 * 2.0 / Ww
    m = ref.silhouette(scr([[4.0, 4.0, 1.0]], Hh, Ww), Hh, Ww, r, 8)[0]
    assert m[4, 4] == 1.0
    w1 = 1.0 - (2.0 / Ww) ** 2 / r ** 2
    for i, j in ((4, 5), (4, 3), (3, 4), (5, 4)):
        assert m[i, j] == pytest.approx(w1, abs=1e-14)
    assert m[4, 6] == pytest.approx(1.0 - 4 * (2.0 / Ww) ** 2 / r ** 2, abs=1e-14)
    assert m[4, 7] == 0.0 and m[1, 4] == 0.0      # 3 pixels away: d2 >= r^2 (strict)
    assert m.sum() > 0 and np.count_nonzero(m) == 21


def test_two_coincident_points():
    Hh = Ww = 9
    r = 2.5 * 2.0 / Ww
    p = [4.3, 4.1, 1.0]
    m1 = ref.silhouette(scr([p], Hh, Ww), Hh, Ww, r, 8)[0]
    m2 = ref.silhouette(scr([p, p[:2] + [2.0]], Hh, Ww), Hh, Ww, r, 8)[0]
    cov = m1 > 0
    np.testing.assert_allclose(m2[cov], 1.0 - (1.0 - m1[cov]) ** 2, atol=1e-14)


def test_only_the_nearest_k_points_count():
    Hh = Ww = 9
    r = 2.5 * 2.0 / Ww
    K = 4
    # K + 3 points around pixel (4, 4), depth decreasing with the index: the kept ones are the LAST K by index
    pts = [[4.5 + 0.25 * k, 4.0 - 0.1 * k, 3.0 - 0.25 * k] for k in range(K + 3)]
    m = ref.silhouette(scr(pts, Hh, Ww), Hh, Ww, r, K)[0]
    w = [1.0 - ((2.0 / Ww) ** 2) * ((q[0] - 4.0) ** 2 + (q[1] - 4.0) ** 2) / r ** 2 for q in pts]
    assert m[4, 4] == pytest.approx(1.0 - np.prod([1.0 - x for x in w[3:]]), abs=1e-14)
    assert abs(m[4, 4] - (1.0 - np.prod([1.0 - x for x in w[:K]]))) > 1e-3
    # equal depths: the lower index wins the last slot
    pts2 = [[4.0 + 0.1 * k, 4.0, 1.0] for k in range(K + 1)]
    P = ref.rasterize(scr(pts2, Hh, Ww), Hh, Ww, r, K)
    at = P["pix"] == 4 * Ww + 4
    assert sorted(P["p"][at].tolist()) == list(range(K))


def test_negative_depth_is_ignored():
    Hh = Ww = 9
    r = 2.5 * 2.0 / Ww
    a = ref.silhouette(scr([[4.2, 3.9, 1.0]], Hh, Ww), Hh, Ww, r, 8)
    b = ref.silhouette(scr([[4.2, 3.9, 1.0], [4.0, 4.0, -0.5]], Hh, Ww), Hh, Ww, r, 8)
    assert np.array_equal(a, b)
    c = ref.silhouette(scr([[4.2, 3.9, 1.0], [4.0, 4.0, 0.0]], Hh, Ww), Hh, Ww, r, 8)
    assert c[0, 4, 4] == 1.0           # Z = 0 is in front of the camera (Z >= 0)


def test_non_square_pixels_are_anisotropic():
    Hh, Ww = 6, 12
    r = 0.5
    m = ref.silhouette(scr([[5.0, 3.0, 1.0]], Hh, Ww), Hh, Ww, r, 8)[0]
    assert m[3, 6] == pytest.approx(1.0 - (2.0 / Ww) ** 2 / r ** 2, abs=1e-14)
    assert m[4, 5] == pytest.approx(1.0 - (2.0 / Hh) ** 2 / r ** 2, abs=1e-14)
    iso = ref.silhouette(scr([[5.0, 3.0, 1.0]], Hh, Ww), Hh, Ww, r, 8, isotropic=True)[0]
    assert iso[4, 5] == pytest.approx(1.0 - (2.0 / Hh) ** 2 / r ** 2, abs=1e-14)
    assert iso[3, 6] == pytest.approx(1.0 - (2.0 / Hh) ** 2 / r ** 2, abs=1e-14)


def test_gradient_matches_central_differences():
    g = np.random.default_rng(3)
    Hh, Ww, K = 10, 14, 3
    r = 0.35
    pts = np.stack([g.uniform(1, Ww - 2, 30), g.uniform(1, Hh - 2, 30), g.uniform(0.5, 2.0, 30)], 1)
    pts[5] = [6.0, 4.0, 0.7]                  # exactly on a pixel centre: a w = 1 factor
    ndc = scr(pts, Hh, Ww)
    G = g.normal(size=(1, Hh, Ww))
    an = ref.silhouette_grad(ndc, Hh, Ww, r, K, G)
    h = 1e-7
    num = np.zeros_like(an)
    for p in range(ndc.shape[1]):
        for a in range(2):
            e = np.zeros_like(ndc)
            e[0, p, a] = h
            num[0, p, a] = ((G * ref.silhouette(ndc + e, Hh, Ww, r, K)).sum()
                            - (G * ref.silhouette(ndc - e, Hh, Ww, r, K)).sum()) / (2 * h)
    err = np.abs(an - num).max() / np.abs(num).max()
    print("restatement gradient vs central differences: max rel %.2e" % err)
    assert err < 1e-6
    # the prod_{q != p} factor matters here
    assert np.abs(ref.silhouette_grad(ndc, Hh, Ww, r, K, G, with_others=False) - num).max() / np.abs(num).max() > 1e-2


def test_hierarchy_switch_installs_builtin_point_renderer(monkeypatch):
    H.dropin()
    from selfreconcode_b200 import synth
    from model.CameraMine import RectifiedPerspectiveCameras
    from model.optim import OptimNetwork
    from model import raster
    monkeypatch.setitem(sys.modules, "pytorch3d", None)        # any pytorch3d import raises
    with pytest.raises(ImportError):
        import pytorch3d  # noqa: F401
    Hh, Ww = 24, 20
    cams = RectifiedPerspectiveCameras(torch.tensor([[20., 20.]]), torch.tensor([[10., 12.]]),
                                       torch.diag(torch.tensor([-1., -1., 1.]))[None], torch.tensor([[0., 0., 2.5]]),
                                       image_size=[(Ww, Hh)])
    ras = raster.MeshRasterizer(cams, raster.RasterSettings((Hh, Ww)))
    net = OptimNetwork(None, None, None, raster.SilhouetteRenderer(ras), None)
    conf = synth.reference_config()
    net.next_conf = conf.get_config('loss_medium')
    net.next_train_conf = conf.get_config('train.medium')
    old_settings = ras.raster_settings
    net.update_hierarchical_config(torch.device("cpu"))
    pr = net.pcRender
    assert isinstance(pr, raster.PointsSilhouetteRenderer) and pr.takes_tensors
    assert pr.radius == conf.get_float('train.medium.point_render.radius')
    s = pr.rasterizer.raster_settings
    assert s.points_per_pixel == 50 and s.image_size == (Hh, Ww)
    assert pr.rasterizer.cameras is cams
    assert isinstance(ras.raster_settings, raster.RasterSettings) and ras.raster_settings is not old_settings
    assert ras.raster_settings.image_size == (Hh, Ww)
    assert net.remesh_intersect == 60 and net.next_conf is None


def test_points_rasterization_settings_defaults():
    H.dropin()
    from model import raster
    s = raster.PointsRasterizationSettings((8, 6))
    assert (s.image_size, s.radius, s.points_per_pixel, s.bin_size) == ((8, 6), 0.01, 8, None)
