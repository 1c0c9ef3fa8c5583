"""CPU: the float64 restatement of the skin-weight volume (tests/lbsw_ref.py) against the reference's own outputs
(boundary.npz: 40 vertices, (7, 9, 5), k = 5, 4 passes) and closed forms, with negative controls that must fail the
fixture's bar."""
import numpy as np
import pytest
import torch

import lbsw_ref as ref
from helpers import golden

BOX = ([-0.6, -0.7, -0.5], [0.6, 0.7, 0.5], (7, 9, 5))
BAR = 2e-6
CUT = 5e-3


def _fixture():
    g = golden("boundary.npz")
    return torch.from_numpy(g["lbsw_verts"]), torch.from_numpy(g["lbsw_ws"]), g


def _err(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def test_restatement_matches_reference_fixture():
    v, w, g = _fixture()
    f, _ = ref.field(*BOX, v, w, 5)
    assert _err(ref.smooth(f, 4, CUT), g["lbsw_field"]) < BAR
    assert _err(ref.smooth(f, 4), g["lbsw_field_model"]) < BAR
    # the renormalisation removes any common scale of the skin weights
    f2, _ = ref.field(*BOX, v, 2 * w, 5)
    assert _err(ref.smooth(f2, 4, CUT), g["lbsw_field"]) < BAR


@pytest.mark.parametrize("name,make", [
    ("gauss_seidel", lambda f: ref.smooth(f, 4, CUT, in_place=True)),
    ("no_renorm", lambda f: ref.smooth(f, 4, CUT, renorm=False)),
    ("cut_every_pass", lambda f: ref.smooth(f, 4, CUT, cut_every_pass=True)),
])
def test_negative_controls_fail_the_bar(name, make):
    """On skin weights scaled by 2 (which the reference's output does not depend on)."""
    v, w, g = _fixture()
    f, _ = ref.field(*BOX, v, 2 * w, 5)
    e = _err(make(f), g["lbsw_field"])
    print("%s: max err %.3e" % (name, e))
    assert e > 100 * BAR


def test_half_voxel_offset_fails_the_bar():
    v, w, g = _fixture()
    f, _ = ref.field(*BOX, v, w, 5, offset=0.5)
    e = _err(ref.smooth(f, 4, CUT), g["lbsw_field"])
    print("centres half a voxel off: max err %.3e" % e)
    assert e > 100 * BAR


def test_k1_without_smoothing_is_the_nearest_vertex():
    v, w, _ = _fixture()
    pts = ref.centres(*BOX)
    f, _ = ref.field(*BOX, v, w, 1)
    near = (pts[:, None, :] - v.double()[None]).norm(dim=-1).argmin(1)
    np.testing.assert_array_equal(f.reshape(24, -1).t().numpy(), w.double()[near].numpy())


def test_vertex_on_a_centre_hits_the_clamp():
    """A vertex exactly on a voxel centre has d = 0 -> weight 1 / 1e-4; a second one 0.5 away weighs 1 / 0.5."""
    pts = torch.tensor([[0.25, 0.0, 0.0]], dtype=torch.float64)
    verts = torch.tensor([[0.25, 0.0, 0.0], [0.25, 0.5, 0.0], [3.0, 3.0, 3.0]], dtype=torch.float64)
    ws = torch.eye(3, dtype=torch.float64)
    d, idx = ref.knn(pts, verts, 2)
    out = ref.blend(d, idx, ws, 2)
    w0, w1 = 1e4, 2.0
    np.testing.assert_allclose(out.numpy(), [[w0 / (w0 + w1), w1 / (w0 + w1), 0.0]], rtol=1e-15)


def test_distance_ties_keep_the_lower_index():
    pts = torch.zeros(1, 3, dtype=torch.float64)
    verts = torch.tensor([[1.0, 0, 0], [0, 0.5, 0], [0, 1.0, 0], [0, 0, -1.0], [-0.5, 0, 0]], dtype=torch.float64)
    d, idx = ref.knn(pts, verts, 3)
    assert idx[0].tolist() == [1, 4, 0, 2]


def test_constant_field_is_invariant_under_a_pass():
    f = torch.full((1, 4, 5, 6, 7), 0.25, dtype=torch.float64)
    np.testing.assert_allclose(ref.smooth(f, 1).numpy(), f.numpy(), rtol=0, atol=1e-16)


def test_impulse_follows_the_stencil():
    """An impulse of 1 at an interior voxel (channel 0; channel 1 is a constant floor): one pass leaves 0.7 there and
    gives each of its six neighbours 0.3 / 6."""
    f = torch.zeros(1, 2, 5, 5, 5, dtype=torch.float64)
    f[0, 1] = 1.0
    f[0, 0, 2, 2, 2] = 1.0
    out = ref.smooth(f, 1, renorm=False)[0, 0]
    assert out[2, 2, 2] == pytest.approx(0.7, abs=1e-15)
    for dz, dy, dx in [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]:
        assert out[2 + dz, 2 + dy, 2 + dx] == pytest.approx(0.3 / 6.0, abs=1e-15)
    assert float(out.sum()) == pytest.approx(0.7 + 0.3, abs=1e-14)


def test_renormalisation_gives_unit_channel_sums():
    g = torch.Generator().manual_seed(0)
    f = torch.rand(1, 7, 4, 5, 6, generator=g, dtype=torch.float64)
    out = ref.smooth(f, 2)
    np.testing.assert_allclose(out.sum(1).numpy(), 1.0, atol=1e-15)
    # a volume with no interior (W = 2) is only renormalised
    f2 = torch.rand(1, 3, 4, 5, 2, generator=g, dtype=torch.float64)
    np.testing.assert_allclose(ref.smooth(f2, 3).numpy(), (f2 / f2.sum(1, keepdim=True)).numpy(), atol=1e-15)
