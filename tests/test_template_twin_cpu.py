"""CPU: the float64 point silhouette the template twin renders with (train_step_twin.Silhouette64 composed with
raster.screen_vertices) passes torch.autograd.gradcheck w.r.t. the vertices and the cameras' inputs on a small scene
away from borderline points, and matches points_silhouette_ref composed with its own K-matrix projection
(project_ndc)."""
import numpy as np
import pytest
import torch
from torch.autograd.gradcheck import GradcheckError

import helpers as H
import points_silhouette_ref as PS
import train_step_twin as TW

Hh, Ww, R_NDC = 14, 16, 0.3


def _scene(seed):
    """Two frames of 12 points, each frame seen by its own camera; K = 3 with more than 3 points on some pixels."""
    g = torch.Generator().manual_seed(seed)
    verts = (torch.randn(2, 12, 3, generator=g, dtype=torch.float64) * 0.12)
    R = torch.diag(torch.tensor([-1., -1., 1.], dtype=torch.float64)).expand(2, 3, 3).clone()
    R[1] = R[1] @ torch.tensor([[np.cos(0.2), 0., np.sin(0.2)], [0., 1., 0.], [-np.sin(0.2), 0., np.cos(0.2)]],
                               dtype=torch.float64)
    T = torch.tensor([[0.02, -0.01, 2.0], [-0.03, 0.02, 2.2]], dtype=torch.float64)
    f = torch.tensor([[40., 38.], [41., 39.]], dtype=torch.float64)
    pp = torch.tensor([[7.6, 6.3], [7.2, 6.6]], dtype=torch.float64)
    return verts, R, T, f, pp


def _render(verts, R, T, f, pp, K):
    H.dropin()
    from model.CameraMine import RectifiedPerspectiveCameras
    from model.raster import screen_vertices
    cams = RectifiedPerspectiveCameras(f, pp, R, T, image_size=[(Ww, Hh)])
    return TW.Silhouette64.apply(screen_vertices(verts, cams), Hh, Ww, R_NDC, K)


def _ndc(verts, R, T, f, pp):
    return PS.project_ndc(verts.numpy(), R.numpy(), T.numpy(), f.numpy(), pp.numpy(), Hh, Ww)


@pytest.mark.parametrize("K", [3, None])
def test_matches_restatement_with_its_own_projection(K):
    verts, R, T, f, pp = _scene(1)
    m = _render(verts, R, T, f, pp, K)[..., 0].numpy()
    ref = PS.silhouette(_ndc(verts, R, T, f, pp), Hh, Ww, R_NDC, K)
    assert (ref > 0).sum() > 40
    np.testing.assert_allclose(m, ref, rtol=0, atol=1e-13)


def test_gradcheck_vertices_and_cameras():
    verts, R, T, f, pp = _scene(1)
    ndc = _ndc(verts, R, T, f, pp)
    assert not PS.borderline_points(ndc, Hh, Ww, R_NDC, 3, rel=1e-4).any()
    assert PS.rasterize(ndc, Hh, Ww, R_NDC, None)["n_cover"].max() > 3      # the K truncation is exercised
    ins = [t.clone().requires_grad_(True) for t in (verts, R, T, f, pp)]
    assert torch.autograd.gradcheck(lambda *a: _render(*a, 3), ins, eps=1e-7, atol=1e-6, rtol=1e-5)


def test_gradcheck_fails_without_the_product_rule(monkeypatch):
    """Negative control: the gradient of the restatement with dmask/dw_p = 1 (no prod_{q != p} (1 - w_q)) is not the
    derivative of its mask, and gradcheck says so."""
    verts, R, T, f, pp = _scene(1)
    grad0 = PS.silhouette_grad

    def no_others(*a, **k):
        return grad0(*a, with_others=False, **k)
    monkeypatch.setattr(PS, "silhouette_grad", no_others)
    v = verts.clone().requires_grad_(True)
    with pytest.raises(GradcheckError):
        torch.autograd.gradcheck(lambda x: _render(x, R, T, f, pp, 3), [v], eps=1e-7, atol=1e-6, rtol=1e-5)
