"""GPU: the skin-weight volume kernels (csrc/lbsw_field.cu) against the float64 restatement (tests/lbsw_ref.py) and the
reference's fixture, and both drop-in compute_lbswField variants on their device path.

Bars: fixture 2e-6 (the CPU test's); blend 1e-5 of float64 on voxels whose k-th and (k+1)-th float64 distances are not
within 1e-5 relative (counted); 30 passes on the device's own blend 2e-6 (values within 1e-6 of the 5e-3 cut counted
and excluded); voxel centres and the (d, index) tie rule bit for bit.  Device outputs are pre-filled with NaN."""
import ctypes as C

import numpy as np
import pytest
import torch

import helpers as H
import lbsw_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
CUT = 5e-3
FULL = (129, 225, 65)


def _lib():
    from selfreconcode_b200 import _lib as L
    return L.load()


def _blend_raw(verts, ws, bmin, bmax, res, k, align=False):
    """sr_lbsw_knn_blend into NaN-filled field / centres buffers."""
    W, H_, D = res
    V, Cc = verts.shape[0], ws.shape[1]
    field = torch.full((1, Cc, D, H_, W), float("nan"), device=DEV)
    cen = torch.full((W * H_ * D, 3), float("nan"), device=DEV)
    lo = (C.c_float * 3)(*[float(x) for x in torch.tensor(bmin, dtype=torch.float32)])
    hi = (C.c_float * 3)(*[float(x) for x in torch.tensor(bmax, dtype=torch.float32)])
    rc = _lib().sr_lbsw_knn_blend(C.c_void_p(verts.data_ptr()), C.c_void_p(ws.data_ptr()), V, Cc, lo, hi, W, H_, D,
                                  int(align), k, C.c_void_p(field.data_ptr()), C.c_void_p(cen.data_ptr()),
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    assert not torch.isnan(field).any() and not torch.isnan(cen).any()
    return field, cen


def _smooth_raw(field, times, cut):
    _, Cc, D, H_, W = field.shape
    src = field.clone()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if times == 0 and cut > 0:
        assert _lib().sr_lbsw_cut(C.c_void_p(src.data_ptr()), src.numel(), cut, stream) == 0
    for t in range(times):
        dst = torch.full_like(src, float("nan"))
        rc = _lib().sr_lbsw_smooth_pass(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), Cc, D, H_, W,
                                        cut if t == times - 1 else 0.0, stream)
        assert rc == 0
        src = dst
    torch.cuda.synchronize()
    assert not torch.isnan(src).any()
    return src


def _voxel_centres(bmin, bmax, res, align=False):
    H.dropin()
    from utils.LBSWsmpl import voxel_centres
    return voxel_centres(bmin, bmax, res, DEV, align)


def _cdist_field(bmin, bmax, res, verts, ws, k, align=False, chunk=50000):
    """The cdist + top-k blend compute_lbswField ran on the device before the kernels existed."""
    W, H_, D = res
    pts = _voxel_centres(bmin, bmax, res, align)
    out = []
    for part in torch.split(pts, chunk):
        dist, idx = torch.cdist(part, verts).topk(k, dim=-1, largest=False)
        w = 1. / dist.clamp(0.0001, 1.)
        w = w / w.sum(-1, keepdim=True)
        out.append((ws[idx.reshape(-1)] * w.reshape(-1, 1)).reshape(w.shape[0], k, -1).sum(1))
    return torch.cat(out, dim=0).transpose(0, 1).reshape(1, -1, D, H_, W)


def _synth_verts(V=6890, C_=24, seed=11, sigma=0.18):
    """V seeded points in the synthetic box with softmax skin weights around the synthetic joints (C_ of them)."""
    from selfreconcode_b200 import synth
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(synth.B_MIN), torch.tensor(synth.B_MAX)
    v = lo + torch.rand(V, 3, generator=g) * (hi - lo)
    J = torch.from_numpy(synth.SYNTH_JOINTS[:C_].copy())
    ws = torch.softmax(-((v[:, None, :] - J[None]) ** 2).sum(-1) / (2 * sigma * sigma), dim=1)
    return v.to(DEV).contiguous(), ws.to(DEV).contiguous(), list(synth.B_MIN), list(synth.B_MAX)


def _check_blend(field, cen, verts, ws, k, res, bar=1e-5):
    """blend vs float64 on the device's own centres; returns (max err, excluded voxels)."""
    f64, d = ref.field(None, None, res, verts, ws, k, pts=cen.double())
    if d.shape[1] > k:
        tie = (d[:, k] - d[:, k - 1]) <= 1e-5 * d[:, k]
    else:
        tie = torch.zeros(d.shape[0], dtype=torch.bool, device=DEV)
    keep = ~tie
    err = (field.double() - f64).abs().reshape(field.shape[1], -1)[:, keep]
    e = float(err.max()) if err.numel() else 0.0
    assert e <= bar, e
    return e, int(tie.sum())


def _check_smooth(field, times, cut):
    """device passes vs float64 passes on the same (device) blend; returns (max err, excluded values)."""
    dev = _smooth_raw(field, times, cut)
    r = ref.smooth(field, times, cut)
    excl = torch.zeros_like(r, dtype=torch.bool)
    if cut > 0:
        excl = (ref.smooth(field, times) - cut).abs() <= 1e-6
    diff = (dev.double() - r).abs()[~excl]
    e = float(diff.max()) if diff.numel() else 0.0
    assert e <= 2e-6, e
    return e, int(excl.sum()), dev


def test_fixture_both_variants():
    H.dropin()
    import utils
    from model.Deformer import compute_lbswField as field_model
    g = H.golden("boundary.npz")
    v, w = torch.from_numpy(g["lbsw_verts"]).to(DEV), torch.from_numpy(g["lbsw_ws"]).to(DEV)
    box = ([-0.6, -0.7, -0.5], [0.6, 0.7, 0.5], (7, 9, 5))
    a = utils.compute_lbswField(*box, v, w, mean_neighbor=5, smooth_times=4)
    b = field_model(*box, v, w, mean_neighbor=5, smooth_times=4)
    ea, eb = np.abs(a.cpu().numpy() - g["lbsw_field"]).max(), np.abs(b.cpu().numpy() - g["lbsw_field_model"]).max()
    print("fixture: utils.LBSWsmpl %.3e, model.Deformer %.3e" % (ea, eb))
    assert ea <= 2e-6 and eb <= 2e-6
    # the public path is the raw kernels
    f, _ = _blend_raw(v, w, *box, 5)
    assert torch.equal(a, _smooth_raw(f, 4, CUT)) and torch.equal(b, _smooth_raw(f, 4, 0.0))


def test_full_size():
    """6 890 vertices, (129, 225, 65), k = 30, 30 passes."""
    H.dropin()
    import utils
    from model.Deformer import compute_lbswField as field_model
    verts, ws, lo, hi = _synth_verts()
    field, cen = _blend_raw(verts, ws, lo, hi, FULL, 30)
    assert torch.equal(cen, _voxel_centres(lo, hi, FULL)), "voxel centres differ from voxel_centres()"
    e, n_tie = _check_blend(field, cen, verts, ws, 30, FULL)
    print("full blend: max err %.3e, %d near-tie voxels excluded of %d" % (e, n_tie, cen.shape[0]))
    e1, _, dev_model = _check_smooth(field, 30, 0.0)
    e2, n_cut, dev_cut = _check_smooth(field, 30, CUT)
    print("full 30 passes: no cut %.3e, cut %.3e (%d values within 1e-6 of the cut excluded)" % (e1, e2, n_cut))
    # public entry points: the same bits, and bit-identical on a rerun
    for _ in range(2):
        assert torch.equal(field_model(lo, hi, FULL, verts, ws, mean_neighbor=30, smooth_times=30), dev_model)
        assert torch.equal(utils.compute_lbswField(lo, hi, FULL, verts, ws, mean_neighbor=30, smooth_times=30),
                           dev_cut)
    old = _cdist_field(lo, hi, FULL, verts, ws, 30)
    print("information: blend vs the cdist path: max |diff| %.3e" % float((old - field).abs().max()))


@pytest.mark.parametrize("k,C_,res,align,times", [
    (1, 24, (33, 41, 17), False, 3),
    (5, 24, (33, 41, 17), True, 3),
    (32, 24, (33, 41, 17), False, 3),
    (30, 7, (33, 41, 17), False, 5),
    (13, 7, (2, 41, 17), False, 4),
    (5, 24, (33, 41, 17), False, 0),
])
def test_shapes(k, C_, res, align, times):
    H.dropin()
    import utils
    verts, ws, lo, hi = _synth_verts(V=1500, C_=C_, seed=5)
    field, cen = _blend_raw(verts, ws, lo, hi, res, k, align)
    assert torch.equal(cen, _voxel_centres(lo, hi, res, align))
    e, n_tie = _check_blend(field, cen, verts, ws, k, res)
    e2, n_cut, dev = _check_smooth(field, times, CUT)
    print("k=%d C=%d res=%s align=%s: blend %.3e (%d ties), %d passes %.3e (%d near cut)" %
          (k, C_, res, align, e, n_tie, times, e2, n_cut))
    assert torch.equal(utils.compute_lbswField(lo, hi, res, verts, ws, align, k, times), dev)


def test_exact_ties_follow_the_index_rule():
    """27 vertices on a 0.5 lattice, voxel centres on the 1/8 lattice i / 8 - 1: distances are exact in fp32 and
    float64 and tie often.  One-hot skin weights expose which vertices each voxel blends: the sets match the restatement's exactly."""
    g = torch.Generator().manual_seed(2)
    lat = torch.stack(torch.meshgrid([torch.tensor([-0.5, 0.0, 0.5])] * 3, indexing="ij"), -1).reshape(-1, 3)
    verts = lat[torch.randperm(27, generator=g)].to(DEV).contiguous()
    ws = torch.eye(27, device=DEV)
    res = (16, 16, 16)
    for k in (1, 5, 8):
        field, cen = _blend_raw(verts, ws, [-1.0625] * 3, [0.9375] * 3, res, k)
        f64, d = ref.field(None, None, res, verts, ws, k, pts=cen.double())
        n_tie = int((d[:, k] == d[:, k - 1]).sum())
        assert torch.equal(field.reshape(27, -1) > 0, f64.reshape(27, -1) > 0)
        assert float((field.double() - f64).abs().max()) <= 1e-6
        print("k=%d: %d voxels with an exact tie at the k-th neighbour" % (k, n_tie))
        assert n_tie > 0


def test_k33_keeps_the_torch_path():
    H.dropin()
    import utils
    verts, ws, lo, hi = _synth_verts(V=800, seed=6)
    res = (17, 21, 9)
    got = utils.compute_lbswField(lo, hi, res, verts, ws, mean_neighbor=33, smooth_times=2)
    want = utils.LBSWsmpl.smooth_weights(_cdist_field(lo, hi, res, verts, ws, 33), 2)
    assert torch.equal(got, want)


def test_invalid_arguments():
    verts, ws, lo, hi = _synth_verts(V=40, seed=1)
    from selfreconcode_b200 import ops
    for kw in (dict(k=0), dict(k=33), dict(k=41)):
        with pytest.raises(RuntimeError):
            ops.lbsw_field(lo, hi, (4, 4, 4), verts, ws, **kw)
    with pytest.raises(RuntimeError):
        ops.lbsw_field(lo, hi, (4, 4, 4), verts, torch.ones(40, 33, device=DEV), k=5)
    with pytest.raises(RuntimeError):
        ops.lbsw_field(lo, hi, (0, 4, 4), verts, ws, k=5)
