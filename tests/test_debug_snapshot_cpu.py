"""CPU: the files of OptimNetwork.save_debug -- the binary PLY writer against an independent parser, and the debug
images' composition against a numpy restatement of the reference's arithmetic (model/network.py:374-447)."""
import os

import numpy as np
import pytest
import torch

import helpers as H


def _snapshot():
    H.dropin()
    from model import snapshot
    return snapshot


def _read_ply(path):
    """A strict parser of the subset write_ply emits: ascii header, binary little-endian float xyz, uchar/int lists."""
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0" and lines[-1] == "end_header"
    nv = nf = None
    props = []
    for ln in lines[2:-1]:
        w = ln.split()
        if w[:2] == ["element", "vertex"]:
            nv = int(w[2])
        elif w[:2] == ["element", "face"]:
            nf = int(w[2])
        elif w[0] == "property":
            props.append(" ".join(w[1:]))
    assert props == ["float x", "float y", "float z", "list uchar int vertex_indices"]
    off = end
    verts = np.frombuffer(data, dtype="<f4", count=nv * 3, offset=off).reshape(nv, 3)
    off += nv * 12
    faces = np.empty((nf, 3), np.int32)
    for i in range(nf):
        assert data[off] == 3
        faces[i] = np.frombuffer(data, dtype="<i4", count=3, offset=off + 1)
        off += 13
    assert off == len(data)
    return verts, faces


@pytest.mark.parametrize("nv,nf", [(5, 4), (7, 0), (1000, 1996)])
def test_ply_round_trip(tmp_path, nv, nf):
    S = _snapshot()
    g = torch.Generator().manual_seed(nv + nf)
    v = torch.randn(nv, 3, generator=g) * 1e3
    v[0] = torch.tensor([float("-0.0"), 1e-40, -3.4e38])        # signed zero, a denormal, a huge value
    f = torch.randint(0, nv, (nf, 3), generator=g)
    if nf:
        f[0] = torch.tensor([0, 0, nv - 1])                      # degenerate rows are written as they are
    path = os.path.join(tmp_path, "m.ply")
    S.write_ply(path, v, f)
    rv, rf = _read_ply(path)
    assert rv.tobytes() == v.numpy().astype("<f4").tobytes()
    assert rf.shape == (nf, 3) and np.array_equal(rf, f.numpy().astype(np.int32))


def test_ply_keeps_duplicate_and_unreferenced_vertices(tmp_path):
    S = _snapshot()
    v = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0., 1., 0.], [0., 0., 0.], [5., 5., 5.]])
    f = torch.tensor([[0, 1, 2], [3, 2, 1]])
    path = os.path.join(tmp_path, "d.ply")
    S.write_ply(path, v, f)
    rv, rf = _read_ply(path)
    assert np.array_equal(rv, v.numpy()) and np.array_equal(rf, f.numpy())


def _seed(N, Hh, Ww, P, g):
    flat = torch.randperm(N * Hh * Ww, generator=g)[:P]
    return flat // (Hh * Ww), (flat // Ww) % Hh, flat % Ww


def test_image_composition_matches_reference_arithmetic():
    S = _snapshot()
    N, Hh, Ww, P = 2, 9, 11, 120
    g = torch.Generator().manual_seed(3)
    bi, ri, ci = _seed(N, Hh, Ww, P, g)
    colors = torch.randn(P, 3, generator=g) * 1.5               # well outside [-1, 1]: clamp + truncation
    colors[:4] = torch.tensor([[-1., 1., 0.], [-1.0000001, 1.0000001, 0.99999994],
                               [-3., 3., 0.5], [0.1, -0.996, 0.]])
    normals = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=1)
    gt = torch.rand(N, Hh, Ww, 3, generator=g) * 2 - 1
    b, r, c = bi.numpy(), ri.numpy(), ci.numpy()
    # numpy restatement of network.py:426-439 in float32
    f32 = np.float32
    tc = np.clip((colors.numpy() / f32(2.) + f32(0.5)) * f32(255.), f32(0.), f32(255.))
    want_rgb = np.full((N, Hh, Ww, 3), 255., np.float32)
    want_rgb[b, r, c] = tc
    want_rgb = want_rgb.astype(np.uint8)
    tn = (normals.numpy() * f32(0.5) + f32(0.5)) * f32(255.)
    want_n = np.full((N, Hh, Ww, 3), 255., np.float32)
    want_n[b, r, c] = tn[:, [2, 1, 0]]
    want_n = want_n.astype(np.uint8)
    want_gt = ((gt.numpy() / f32(2.) + f32(0.5)) * f32(255.)).astype(np.uint8)
    rgb = S.color_image(colors, bi, ri, ci, gt)
    nimg = S.normal_image(normals, bi, ri, ci, gt)
    gimg = S.gt_color_image(gt)
    assert rgb.dtype == nimg.dtype == gimg.dtype == np.uint8
    assert np.array_equal(rgb, want_rgb) and np.array_equal(nimg, want_n) and np.array_equal(gimg, want_gt)
    # the clamp and the truncating cast were both exercised
    assert (want_rgb[b, r, c] == 0).any() and (want_rgb[b, r, c] == 255).any()
    assert rgb[b[3], r[3], c[3], 0] == 140         # (0.1/2+0.5)*255 = 140.25 truncates
    covered = np.zeros((N, Hh, Ww), bool)
    covered[b, r, c] = True
    assert np.all(rgb[~covered] == 255) and np.all(nimg[~covered] == 255)


def test_mask_image():
    S = _snapshot()
    m = torch.tensor([[[0., 0.5, 1.], [0.999, 0.0039, 1.0001]]])[..., None]
    assert np.array_equal(S.mask_image(m)[..., 0], np.array([[[0, 127, 255], [254, 0, 255]]], np.uint8))
