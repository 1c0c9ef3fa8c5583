"""CPU: PLY reading, OBJ writing, the chart packer and closed forms of the float64 twin (tests/uvmap_ref.py)."""
import os

import numpy as np
import pytest
import torch

import helpers  # noqa: F401  (puts the repository root on sys.path)
from selfreconcode_b200 import uvmap, texture
import uvmap_ref as U

V4 = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32)
F2 = np.array([[0, 1, 2], [0, 2, 3]], np.int64)


def _write(path, text, body=b""):
    with open(path, "wb") as fh:
        fh.write(text.encode("ascii") + body)


def test_read_openmesh_ascii(tmp_path):
    p = str(tmp_path / "tmp.ply")
    _write(p, "ply\nformat ascii 1.0\ncomment made by OpenMesh\nelement vertex 4\nproperty float x\nproperty float y\n"
              "property float z\nelement face 2\nproperty list uchar int vertex_indices\nend_header\n"
              "0 0 0\n1 0 0\n1 1 0\n0 1 0\n3 0 1 2\n3 0 2 3\n")
    V, F = uvmap.read_mesh(p)
    assert V.dtype == torch.float32 and F.dtype == torch.int64
    assert np.array_equal(V.numpy(), V4) and np.array_equal(F.numpy(), F2)


def test_read_snapshot_write_ply(tmp_path):
    helpers.dropin()
    from model.snapshot import write_ply
    g = np.random.default_rng(0)
    V = g.standard_normal((50, 3)).astype(np.float32)
    F = g.integers(0, 50, (80, 3))
    p = str(tmp_path / "s.ply")
    write_ply(p, torch.from_numpy(V), torch.from_numpy(F))
    V2, F2_ = uvmap.read_mesh(p)
    assert np.array_equal(V2.numpy(), V) and np.array_equal(F2_.numpy(), F)


def test_read_double_uint_with_extra_properties_and_quad(tmp_path):
    vdt = np.dtype([("nx", "<f4"), ("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("red", "u1")])
    v = np.zeros(4, vdt)
    v["x"], v["y"], v["z"] = V4[:, 0], V4[:, 1], V4[:, 2]
    face = np.array([4], "<u4").tobytes() + np.array([0, 1, 2, 3], "<u4").tobytes()
    p = str(tmp_path / "d.ply")
    _write(p, "ply\nformat binary_little_endian 1.0\nelement vertex 4\nproperty float nx\nproperty double x\n"
              "property double y\nproperty double z\nproperty uchar red\nelement face 1\n"
              "property list uint uint vertex_indices\nend_header\n", v.tobytes() + face)
    V, F = uvmap.read_mesh(p)
    assert np.array_equal(V.numpy(), V4) and np.array_equal(F.numpy(), F2)


@pytest.mark.parametrize("header", [
    "ply\nformat binary_big_endian 1.0\nelement vertex 0\nproperty float x\nproperty float y\nproperty float z\n"
    "element face 0\nproperty list uchar int vertex_indices\nend_header\n",
    "ply\nformat ascii 1.0\nelement vertex 0\nproperty float x\nproperty float y\n"
    "element face 0\nproperty list uchar int vertex_indices\nend_header\n",
    "ply\nformat ascii 1.0\nelement vertex 0\nproperty float x\nproperty float y\nproperty float z\n"
    "element face 0\nproperty list uchar float vertex_indices\nend_header\n",
    "ply\nformat ascii 1.0\nelement vertex 0\nproperty float x\nproperty float y\nproperty float z\n",
    "obj\n",
])
def test_read_rejects_malformed(tmp_path, header):
    p = str(tmp_path / "bad.ply")
    _write(p, header)
    with pytest.raises(ValueError, match="bad.ply"):
        uvmap.read_mesh(p)


def test_write_obj_round_trip_is_exact(tmp_path):
    g = np.random.default_rng(1)
    V = (g.standard_normal((30, 3)) * 10).astype(np.float32)
    vt = g.random((40, 2)).astype(np.float32)
    F, ft = g.integers(0, 30, (20, 3)), g.integers(0, 40, (20, 3))
    p = str(tmp_path / "template" / "uvmap.obj")
    uvmap.write_obj(p, V, F, vt, ft)
    V2, F2_, vt2, ft2 = texture.load_obj_uv(p)
    assert np.array_equal(V2.numpy(), V) and np.array_equal(vt2.numpy(), vt)
    assert np.array_equal(F2_.numpy(), F) and np.array_equal(ft2.numpy(), ft)


@pytest.mark.parametrize("seed", range(4))
def test_packer(seed):
    g = np.random.default_rng(seed)
    n = int(g.integers(1, 200))
    box = g.random((n, 2)) * np.array([3.0, 1.0]) + 1e-3
    box.sort(1)
    box = box[:, ::-1].copy()          # landscape, as the projection leaves them
    R, pad = 512, 4
    offs, s = uvmap.pack_charts(box, R, pad)
    offs2, s2 = uvmap.pack_charts(box, R, pad)
    assert np.array_equal(offs, offs2) and s == s2
    lo, hi = offs, offs + box * s
    g_ = pad / R
    assert (lo >= g_ - 1e-12).all() and (hi <= 1 - g_ + 1e-12).all()
    for i in range(n):
        for j in range(i + 1, n):
            gap = max(lo[j, 0] - hi[i, 0], lo[i, 0] - hi[j, 0], lo[j, 1] - hi[i, 1], lo[i, 1] - hi[j, 1])
            assert gap >= g_ - 1e-12, (i, j, gap)
    # the scale is the largest that fits, to the bisection's resolution
    assert uvmap.pack_charts(box * (1 + 1e-6), R, pad)[1] <= s


def test_twin_unit_square_quadric():
    Q = U.face_quadric(*V4[[0, 1, 2]].astype(np.float64)) + U.face_quadric(*V4[[0, 2, 3]].astype(np.float64))
    expect = np.zeros((4, 4))
    expect[2, 2] = 1.0             # plane z = 0, total area 1
    assert np.allclose(Q, expect, atol=1e-15)


def test_twin_coplanar_fan_costs_zero():
    ang = np.linspace(0, 2 * np.pi, 7)[:-1]
    V = np.concatenate([[[0, 0, 0]], np.stack([np.cos(ang), np.sin(ang), 0 * ang], 1)]).astype(np.float64)
    F = np.array([[0, 1 + i, 1 + (i + 1) % 6] for i in range(6)])
    Q = U.quadrics(V, F)
    for b in range(1, 7):
        v, c, solved = U.solve(Q[0] + Q[b], V[0], V[b])
        assert c == 0.0 and not solved
        assert np.array_equal(v, V[0])


def test_twin_link_condition_rejects_tetrahedron():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64)
    F = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    fixed = U.fixed_vertices(F, 4)
    assert not fixed.any()
    for a, b in U.edges(F):
        ok, _ = U.edge_checks(V, F, a, b, 0.5 * (V[a] + V[b]), fixed)
        assert not ok


def test_twin_fixed_vertices():
    # a square (all boundary) and two tetrahedra sharing vertex 0
    assert U.fixed_vertices(F2, 4).all()
    T = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    two = np.concatenate([T, np.where(T == 0, 0, T + 3)])
    fx = U.fixed_vertices(two, 7)
    assert fx[0] and not fx[1:].any()
