"""GPU: the tensor-core surface tracer (ops._trace_surface_points_tc, csrc/trace_tc.cu) against float64 restatements.

  * its pointwise stages through the raw C ABI, on their own fp32 inputs, into sentinel-filled buffers: sr_tc_embed
    with an active list, sr_tc_trace_mid, sr_tc_trace_update and sr_tc_render_embed.  Each runs with no list, a
    permutation, a shuffled strict subset and an empty list (m_dev = 0), at 1, 127, 128 and 129 rows (either side of
    the 128-row tile) and at a count past the kernel's first grid-stride wave.  The stages index some buffers by list
    position i and others by global ray gp; only a list that is not the identity tells the two apart;
  * whole traces at the production networks against oracle.optimize_surface_ps in float64, with the rays whose
    decisions lie within the engine's error bounds marked sensitive and excluded;
  * invariances, bitwise: permutation, prefix, rerun (through the CUDA graph), dual- against single-stream sweeps, and
    graph replays after the contents (pose, latent codes, batch indices, rays, start points) change.

Every measured maximum is printed beside its bar (pytest -s)."""
import ctypes as C
import math

import pytest
import torch

import ffma_ref as R
from helpers import elem_err
from oracle import oracle as O
from test_gpu_ffma_contract import (ATHR, CAM, CONDLEN, ELEM, NFRAMES, PAD, SENT, _invariant, _lib, _oracle_trace, _p,
                                    _s, _sample, _split_threshold, _trace_setup, conds, lbs_keep, lbs_setup, report,
                                    sentinel, untouched)

pytestmark = pytest.mark.gpu

NSM = 132
WAVE_WARP = NSM * 8 * 256 // 32     # sr_grid_for caps a grid at 8 CTAs of 256 threads per SM: a warp per ray wraps here
WAVE_THREAD = NSM * 8 * 256         # ... and a thread per ray (or per element) here
# sincosf is within 2 ulp of the result; with the band weight's product, 4 ulp of |ref| plus a floor for values at 0
SIN_TOL = 2.0 ** -21
LD_TRACE = 32                       # the tracer's cotangent row width (_tc_trace_body)


def _lists(P, dev, seed):
    """Active-list cases: (name, index or None, m_dev or None, global ids of the listed rows in list order).  The
    subset's index array is a whole permutation: rows past m_dev name other rays, which no kernel may touch."""
    g = torch.Generator().manual_seed(seed)
    perm = torch.randperm(P, generator=g)
    cases = [("identity", None, None, torch.arange(P)), ("permutation", perm, P, perm)]
    m = (2 * P) // 3
    if 0 < m < P:
        sub = torch.randperm(P, generator=g)
        cases.append(("subset %d" % m, sub, m, sub[:m]))
    cases.append(("empty", torch.randperm(P, generator=g), 0, perm[:0]))
    return [(name, idx.int().to(dev) if idx is not None else None,
             torch.tensor([m], dtype=torch.int32, device=dev) if m is not None else None, ids.to(dev))
            for name, idx, m, ids in cases]


def _pw(ws):
    return (C.c_float * 16)(*(list(ws) + [0.0] * (16 - len(ws))))


def _pad32(n):
    return (n + 31) // 32 * 32


def _sincos_check(name, got, ref, w_cols):
    """PE columns within sincosf's error: |got - ref| <= SIN_TOL (|ref| + w / 32); exactly 0 in a band of weight 0."""
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    tol = SIN_TOL * (ref.abs() + w_cols.view(1, -1) / 32)
    zero = (w_cols == 0).view(1, -1).expand_as(err)
    assert bool((got[zero] == 0).all()), name
    worst = float((err[~zero] / tol[~zero]).max()) if err[~zero].numel() else 0.0
    print("  %-40s max |err| %.2e  (%.2f of the sincosf bar)" % (name, float(err.max()) if err.numel() else 0.0, worst))
    assert worst <= 1.0, name


def _pe_weights_per_column(pw, multires):
    return torch.tensor([pw[b] for b in range(multires) for _ in range(6)], dtype=torch.float64)


# ---------------------------------------------------------------------------------------------------------------------
# sr_tc_embed with an active list (ch = 1: the tracer's forward sweeps)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", ["sdf", "translator"])
def test_embed_active_list_matches_fp64(cuda_dev, net):
    """Row i embeds pts[index[i]] (the translator also appends conds[batch_inds[index[i]]] bit for bit), padding
    columns up to ld are 0, and rows i >= m_dev are not written: the kernel's total is m_dev rows."""
    lib = _lib()
    mr, pw = 6, R.annealing_weights(6, 0.8)
    assert 0.0 in pw and any(0.0 < w < 1.0 for w in pw), "the band weights must include a zero and a fraction"
    cd = conds(cuda_dev) if net == "translator" else None
    condlen = CONDLEN if cd is not None else 0
    pe = 3 + 6 * mr
    ld = _pad32(pe + condlen)
    sizes = (1, 127, 128, 129, WAVE_THREAD // 64 + 3)      # the last wraps the grid at either width
    Pmax = sizes[-1]
    pts_all = _sample(Pmax, 31, -1.3, 1.3).to(cuda_dev)
    bi_all = torch.randint(0, NFRAMES, (Pmax,), generator=torch.Generator().manual_seed(32)).to(cuda_dev)
    e64_all = R.embed(pts_all, mr, pw)
    wcol = _pe_weights_per_column(pw, mr).to(cuda_dev)
    print("embed %s: ld %d" % (net, ld))
    for P in sizes:
        pts, bi = pts_all[:P].contiguous(), bi_all[:P].contiguous()
        for name, idx, m_dev, ids in _lists(P, cuda_dev, P + 1):
            M = ids.numel()
            out = sentinel(P * ld, cuda_dev)
            assert lib.sr_tc_embed(_p(pts), P, mr, _pw(pw), 1, _p(cd), _p(bi), 0, condlen, _p(out), ld, _p(idx),
                                   _p(m_dev), _s()) == 0
            torch.cuda.synchronize()
            assert untouched(out, M * ld), ("rows past m_dev", P, name)
            o = out[:M * ld].view(M, ld)
            assert torch.equal(o[:, :3], pts[ids]), ("points", P, name)
            _sincos_check("PE P=%d %s" % (P, name), o[:, 3:pe], e64_all[ids][:, 3:], wcol)
            if condlen:
                assert torch.equal(o[:, pe:pe + condlen], cd[bi[ids]]), ("conditioning columns", P, name)
            assert bool((o[:, pe + condlen:] == 0).all()), ("padding columns", P, name)


# ---------------------------------------------------------------------------------------------------------------------
# sr_tc_trace_mid
# ---------------------------------------------------------------------------------------------------------------------
DTH = 1e-3
ANG_BAND = 2e-5      # relative: a float32 angle is this close to athreshold only by rounding


def _trace_params(dth, athr):
    from selfreconcode_b200._lib import TraceParams
    tp = TraceParams()
    tp.cam_pos[:] = list(CAM)
    tp.dthreshold, tp.athreshold, tp.w1, tp.w2 = dth, athr, 3.05, 1.0
    return tp


def _mid_inputs(P, with_off, st, lref, dev, seed):
    """Per global ray: start point, translator offset, batch index, f; D(p + off) and M = dD/dp' in float64, and a ray
    at a chosen angle from D - cam: well inside, well outside and within 0.1 % of athreshold."""
    g = torch.Generator().manual_seed(seed)
    pts = _sample(P, seed, -0.7, 0.7).to(dev)
    off = (0.02 * torch.randn(P, 3, generator=g)).to(dev) if with_off else None
    bi = torch.randint(0, NFRAMES, (P,), generator=g).to(dev)
    # f: both signs, exact zeros, dthreshold itself and its float32 neighbours
    f = (DTH * 3 * (2 * torch.rand(P, generator=g) - 1)).float()
    k = torch.randint(0, 8, (P,), generator=g)
    dth32 = torch.tensor(DTH, dtype=torch.float32)
    near = torch.stack([torch.zeros(()), dth32, torch.nextafter(dth32, torch.tensor(1.0)),
                        torch.nextafter(dth32, torch.tensor(0.0))])
    sign = torch.where(torch.rand(P, generator=g) < 0.5, -1.0, 1.0)
    f = torch.where(k < 4, sign * near[k.clamp(max=3)], f).to(dev)
    p1 = pts.double() + (off.double() if off is not None else 0.0)
    if st is not None:
        A, trans = st.A.double(), st.trans.double()      # the kernel's own bone transforms
        bmin = torch.tensor(list(st.params.bmin), dtype=torch.float64, device=dev)
        bmax = torch.tensor(list(st.params.bmax), dtype=torch.float64, device=dev)
        D, Mj = R.jacobian(lambda x: O.lbs_forward(lref["ws"], bmin, bmax, A, trans, x, bi), p1)
        smooth = lbs_keep(lref, p1)[0]
    else:
        D, Mj = p1, torch.eye(3, dtype=torch.float64, device=dev).expand(P, 3, 3)
        smooth = torch.ones(P, dtype=torch.bool, device=dev)
    cam = torch.tensor(CAM, dtype=torch.float64, device=dev)
    u = D - cam
    uh = u / u.norm(dim=1, keepdim=True)
    r = torch.randn(P, 3, generator=g, dtype=torch.float64).to(dev)
    w = r - (r * uh).sum(1, keepdim=True) * uh
    w = w / w.norm(dim=1, keepdim=True)
    factor = torch.tensor([0.3, 0.7, 0.999, 1.001, 1.5, 3.0], dtype=torch.float64)[
        torch.randint(0, 6, (P,), generator=g)].to(dev)
    th = math.radians(ATHR) * factor
    rays = (torch.cos(th).view(-1, 1) * uh + torch.sin(th).view(-1, 1) * w).float()
    return pts, off, bi, f, D, Mj, smooth, rays


def _mid_fp64(D, Mj, rays, f, tp):
    """ray test, loss = w1 |f| + w2 sin and u = w2 M^T d sin / d u in float64, per global ray."""
    cam = torch.tensor(list(tp.cam_pos), dtype=torch.float64, device=D.device)
    uu = (D - cam).detach().requires_grad_(True)
    v = rays.double()
    s = torch.cross(uu, v, dim=1).norm(dim=1) / uu.norm(dim=1)
    (q,) = torch.autograd.grad(s.sum(), uu)
    s = s.detach()
    ang = torch.rad2deg(torch.asin(s))
    done = (f.double().abs() < tp.dthreshold) & (ang < tp.athreshold)
    loss = tp.w1 * f.double().abs() + tp.w2 * s
    u = tp.w2 * torch.einsum("pij,pi->pj", Mj, q)
    u_scale = tp.w2 * torch.einsum("pij,pi->pj", Mj.abs(), q.abs())     # what the float32 dot products round
    near = (ang - tp.athreshold).abs() < ANG_BAND * tp.athreshold
    return done, loss, u, u_scale, near


@pytest.mark.parametrize("with_off,with_lbs", [(True, True), (False, True), (True, False), (False, False)])
def test_trace_mid_matches_fp64(cuda_dev, with_off, with_lbs):
    lib = _lib()
    st, lref = lbs_setup(cuda_dev) if with_lbs else (None, None)
    tp = _trace_params(DTH, ATHR)
    ld = LD_TRACE
    excluded = total = 0
    print("trace_mid off=%d lbs=%d" % (with_off, with_lbs))
    for P in (1, 127, 128, 129, WAVE_WARP + 3):
        pts, off_g, bi, f_g, D, Mj, smooth, rays = _mid_inputs(P, with_off, st, lref, cuda_dev, 40 + P)
        done, loss64, u64, u_scale, near = _mid_fp64(D, Mj, rays, f_g, tp)
        g = torch.Generator().manual_seed(P)
        for name, idx, m_dev, ids in _lists(P, cuda_dev, P + 2):
            M = ids.numel()
            # rows hold the values of their listed ray; rows past m_dev hold other rays' values
            rest = torch.randperm(P, generator=g).to(cuda_dev)
            rows = torch.cat([ids, rest[:P - M]])
            f_rows = f_g[rows].contiguous()
            off_rows = off_g[rows].contiguous() if off_g is not None else None
            listed = torch.zeros(P, dtype=torch.bool, device=cuda_dev)
            listed[ids] = True
            for do_update in (0, 1):
                conv0 = torch.full((P + PAD,), 0xA5, dtype=torch.uint8, device=cuda_dev)
                conv0[:P][listed] = torch.randint(0, 2, (P,), generator=g, dtype=torch.uint8).to(cuda_dev)[listed]
                conv = conv0.clone()
                dsdf, ddef, aux = sentinel(P * ld, cuda_dev), sentinel(P * ld, cuda_dev), sentinel(P * 8, cuda_dev)
                assert lib.sr_tc_trace_mid(_p(idx), _p(m_dev), P, _p(pts), _p(rays), _p(bi), _p(f_rows),
                                           _p(off_rows), C.byref(st.params) if st is not None else None,
                                           C.byref(tp), do_update, _p(conv), _p(dsdf),
                                           _p(ddef) if with_off else None, ld, _p(aux), _s()) == 0
                torch.cuda.synchronize()
                tag = "P=%d %s upd=%d" % (P, name, do_update)
                # flags: set exactly where the float64 test passes, never cleared, unlisted rays untouched
                dec = ~near[ids]
                want = conv0[:P].clone()
                want[ids[done[ids]]] = 1
                assert torch.equal(conv[P:], conv0[P:]), ("padding flags", tag)
                assert torch.equal(conv[:P][~listed], conv0[:P][~listed]), ("unlisted flags", tag)
                assert torch.equal(conv[ids][dec], want[ids][dec]), ("flags", tag)
                assert bool((conv[ids][conv0[ids] == 1] == 1).all()), ("flags already set stay set", tag)
                excluded += int((~dec).sum())
                total += M
                # aux: loss, state, u; its columns 5..7 and the rows past M are not written
                a = aux[:P * 8].view(P, 8)
                assert untouched(aux, P * 8) and bool((a[:, 5:].view(torch.int32) == SENT).all())
                assert bool((a[M:].view(torch.int32) == SENT).all()), ("aux rows past M", tag)
                a = a[:M]
                state = a[:, 1].view(torch.int32)
                state64 = (~done[ids] & bool(do_update)).int()
                assert torch.equal(state[dec], state64[dec]), ("state", tag)
                upd = (state == 1)
                assert bool((a[~upd][:, 0] == 0).all()) and bool((a[~upd][:, 2:5] == 0).all()), ("state-0 rows", tag)
                if int(upd.sum()):
                    report("loss " + tag, a[upd][:, 0], loss64[ids][upd], True)
                    # u = w2 M^T q: each component is a float32 dot product, so its error is relative to the sum of
                    # its terms' magnitudes (M carries the skinning grid's float32 derivative)
                    sm = smooth[ids][upd]
                    ug, ur, us = a[upd][:, 2:5][sm].double(), u64[ids][upd][sm], u_scale[ids][upd][sm]
                    if ur.numel():
                        eu = float(((ug - ur).abs() / (us + ur.abs().mean())).max())
                        print("  %-40s elem (of the terms) %.2e" % ("u " + tag, eu))
                        assert eu < ELEM, ("u", tag, eu)
                # cotangent rows: w1 sign(f) in column 0 of state-1 rows, u in columns 0..2 of ddef, zeros elsewhere
                ds = dsdf[:P * ld].view(P, ld)
                assert bool((ds[M:].view(torch.int32) == SENT).all()) and untouched(dsdf, P * ld), ("dsdf rows", tag)
                w1 = torch.tensor(tp.w1, dtype=torch.float32, device=cuda_dev)
                c0 = torch.where(upd, w1 * torch.sign(f_rows[:M]), torch.zeros_like(f_rows[:M]))
                assert torch.equal(ds[:M, 0], c0), ("dsdf column 0", tag)
                assert bool((ds[:M, 1:] == 0).all()), ("dsdf columns 1..", tag)
                if with_off:
                    dd = ddef[:P * ld].view(P, ld)
                    assert bool((dd[M:].view(torch.int32) == SENT).all()) and untouched(ddef, P * ld), ("ddef", tag)
                    assert torch.equal(dd[:M, :3], a[:, 2:5]), ("ddef columns 0..2", tag)
                    assert bool((dd[:M, 3:] == 0).all()), ("ddef columns 3..", tag)
    print("  %d of %d listed rays within float32 rounding of athreshold, excluded" % (excluded, total))
    assert excluded <= max(2, total // 500)


# ---------------------------------------------------------------------------------------------------------------------
# sr_tc_trace_update
# ---------------------------------------------------------------------------------------------------------------------
PW_S = R.annealing_weights(6, 1.0)      # sdfRatio 1.0
PW_D = R.annealing_weights(6, 0.8)      # deformerRatio 0.8


@pytest.mark.parametrize("with_skip,with_def", [(True, True), (False, True), (True, False), (False, False)])
def test_trace_update_matches_fp64(cuda_dev, with_skip, with_def):
    """p <- x - loss / |g|^2 g with g = u + (d embed_s / dx)^T (gs + gskip) + (d embed_d / dx)^T gd; state-0 and
    unlisted rays bit-unchanged; the appended list is exactly the updated rays, and nothing past its count is
    written."""
    lib = _lib()
    mr, pe = 6, 39
    print("trace_update skip=%d translator=%d" % (with_skip, with_def))
    for P in (1, 127, 128, 129, WAVE_THREAD + 3):
        g = torch.Generator().manual_seed(50 + P)
        x = _sample(P, 60 + P, -1.0, 1.0).to(cuda_dev)
        gs = (0.5 * torch.randn(P, 64, generator=g)).to(cuda_dev)
        gk = (0.5 * torch.randn(P, 64, generator=g)).to(cuda_dev) if with_skip else None
        gd = (0.5 * torch.randn(P, 64, generator=g)).to(cuda_dev) if with_def else None
        aux = torch.randn(P, 8, generator=g)
        # losses that make steps of ~0.1: a step read back as p - x carries p's float32 rounding
        aux[:, 0] = 1.0 + 4.0 * torch.rand(P, generator=g)
        aux[:, 2:5] *= 0.3
        state = (torch.rand(P, generator=g) < 0.75).int()
        aux = aux.to(cuda_dev)
        aux[:, 1] = state.to(cuda_dev).view(torch.float32)
        for name, idx, m_dev, ids in _lists(P, cuda_dev, P + 3):
            M = ids.numel()
            tag = "P=%d %s" % (P, name)
            pts = sentinel(P * 3, cuda_dev)
            pts[:P * 3] = x.view(-1)
            act = torch.full((P + PAD,), SENT, dtype=torch.int32, device=cuda_dev)
            counter = torch.zeros(1, dtype=torch.int32, device=cuda_dev)
            assert lib.sr_tc_trace_update(_p(idx), _p(m_dev), P, _p(pts), _p(gs), 64, _p(gk), 64, _p(gd),
                                          64 if with_def else 0, _p(aux), mr, _pw(PW_S), mr if with_def else 0,
                                          _pw(PW_D) if with_def else None, _p(act), _p(counter), _s()) == 0
            torch.cuda.synchronize()
            rows = torch.nonzero(aux[:M, 1].view(torch.int32) == 1).view(-1)
            gp = ids[rows]
            n = int(counter)
            assert n == gp.numel(), ("counter", tag)
            assert torch.equal(act[:n].sort().values, gp.int().sort().values), ("appended list", tag)
            assert bool((act[n:] == SENT).all()), ("list past its count", tag)
            assert untouched(pts, P * 3)
            out = pts[:P * 3].view(P, 3)
            moved = torch.zeros(P, dtype=torch.bool, device=cuda_dev)
            moved[gp] = True
            assert torch.equal(out[~moved].view(torch.int32), x[~moved].view(torch.int32)), ("unchanged rays", tag)
            if not gp.numel():
                continue
            xd = x[gp].double().requires_grad_(True)
            cot = gs[rows, :pe].double() + (gk[rows, :pe].double() if gk is not None else 0.0)
            obj = (R.embed(xd, mr, PW_S) * cot).sum()
            if gd is not None:
                obj = obj + (R.embed(xd, mr, PW_D) * gd[rows, :pe].double()).sum()
            (gx,) = torch.autograd.grad(obj, xd)
            gv = gx + aux[rows, 2:5].double()
            loss = aux[rows, 0].double()
            step = -(loss / (gv * gv).sum(1)).view(-1, 1) * gv
            # g is a float32 sum of the chain's terms: its error is relative to their magnitudes, and a step's to
            # that over |g| (a ray whose terms cancel is that much worse conditioned)
            xs = xd.detach()
            scale = aux[rows, 2:5].double().abs() + _chain_scale(xs, cot, PW_S)
            if gd is not None:
                scale += _chain_scale(xs, gd[rows, :pe].double(), PW_D)
            kappa = (scale.norm(dim=1) / gv.norm(dim=1)).clamp(min=1.0)
            es = float(((out[gp].double() - x[gp].double() - step).norm(dim=1) / step.norm(dim=1) / kappa).max())
            print("  %-40s step rel. err / conditioning %.2e (conditioning up to %.1f)"
                  % ("step " + tag, es, float(kappa.max())))
            assert es < ELEM, ("step", tag, es)
            report("points " + tag, out[gp], xs + step, True)


def _chain_scale(x, cot, pw):
    """Per coordinate: the sum of the magnitudes of the terms of (d embed / dx)^T cot."""
    s = cot[:, :3].abs()
    for b in range(len(pw)):
        fr = 2.0 ** b
        s = s + pw[b] * fr * ((torch.cos(x * fr) * cot[:, 3 + 6 * b:6 + 6 * b]).abs()
                              + (torch.sin(x * fr) * cot[:, 6 + 6 * b:9 + 6 * b]).abs())
    return s


# ---------------------------------------------------------------------------------------------------------------------
# sr_tc_render_embed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stride,col0", [(1, 1), (4, 0), (4, 3)])
def test_render_embed_matches_fp64(cuda_dev, stride, col0):
    """cat(points, PE(view), normals, features): copies bit for bit, the view's encoding within sincosf's error,
    zeros up to ld, nothing past P rows."""
    lib = _lib()
    mr, nfeat = 4, 256
    pw = R.annealing_weights(mr, 0.6)
    assert 0.0 in pw and any(0.0 < w < 1.0 for w in pw)
    pe = 3 + 6 * mr
    ld = _pad32(3 + pe + 3 + nfeat)
    feat_ld = col0 + nfeat + 5
    wcol = _pe_weights_per_column(pw, mr).to(cuda_dev)
    print("render_embed stride %d col0 %d: ld %d" % (stride, col0, ld))
    for P in (1, 127, 128, 129, WAVE_THREAD // ld + 3):
        g = torch.Generator().manual_seed(70 + P)
        pts = torch.randn(P, 3, generator=g).to(cuda_dev)
        views = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=1).to(cuda_dev)
        nrm = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=1).to(cuda_dev)
        feat = torch.randn(P * stride, feat_ld, generator=g).to(cuda_dev)
        out = sentinel(P * ld, cuda_dev)
        assert lib.sr_tc_render_embed(P, _p(pts), _p(views), _p(nrm), _p(feat), feat_ld, col0, nfeat, stride, mr,
                                      _pw(pw), _p(out), ld, _s()) == 0
        torch.cuda.synchronize()
        assert untouched(out, P * ld)
        o = out[:P * ld].view(P, ld)
        assert torch.equal(o[:, :3], pts) and torch.equal(o[:, 3:6], views)
        _sincos_check("view PE P=%d" % P, o[:, 6:3 + pe], R.embed(views, mr, pw)[:, 3:], wcol)
        assert torch.equal(o[:, 3 + pe:6 + pe], nrm)
        assert torch.equal(o[:, 6 + pe:6 + pe + nfeat], feat[::stride][:, col0:col0 + nfeat])
        assert bool((o[:, 6 + pe + nfeat:] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# whole tensor-core traces against oracle.optimize_surface_ps in float64 (on the GPU)
# ---------------------------------------------------------------------------------------------------------------------
# (sdf, translator, LBS) and a ray count at a tile edge; mode "tc" is forced below ops.TC_MIN_POINTS
TC_PAIRS = {
    "translator_lbs": (("ref_sdf", "translator_ref", True), 2433),      # 19 tiles + 1 row
    "translator": (("ref_sdf", "translator_ref", False), 1151),         # 9 tiles - 1 row
    "identity": (("ref_sdf", None, False), 640),                        # 5 whole tiles
    "lbs": (("ref_sdf", None, True), 383),                              # 3 tiles - 1 row: off = NULL with LBS
}


# The translator's ReLU units switch where their pre-activation crosses 0, and with them d offset / dp.  The fp32 engine
# decides them within 1e-5 (test_gpu_ffma_contract.RELU_MARGIN); the tensor-core engine's error on f is 20 times the
# fp32 engine's (TC_EPS_F against 2e-6), and so is this margin.
RELU_MARGIN_TC = 2e-4


def _kink_free(dnet, cd, cam, rays, x0, bi, sdf_fn, def_fn, dth, times, iters):
    """Rays whose float64 trajectory keeps every ReLU pre-activation of the translator farther than RELU_MARGIN_TC
    from 0 at each point where a Newton step takes its gradient."""
    keep = torch.ones(x0.shape[0], dtype=torch.bool, device=x0.device)
    if dnet is None:
        return keep
    for k in range(times):
        xk = x0 if k == 0 else _oracle_trace(cam, rays, x0, bi, sdf_fn, def_fn, dth, k)[0]
        with torch.no_grad():
            _, zs = R.translator_offset(dnet.layers, xk, 6, dnet.pe_w, cd, bi, with_preacts=True)
        keep &= (R.min_relu_margin(dnet.layers, zs) >= RELU_MARGIN_TC) | (iters <= k)
    return keep


def _tc_trace(sdf, dnet, st, cd, x0, rays, bi, dth, times):
    from selfreconcode_b200 import ops
    dev = sdf.fused.device
    return ops.trace_surface_points(sdf.fused.truncated_last(1), dnet.fused if dnet else None, st,
                                    torch.tensor(CAM, device=dev), rays.float().to(dev), x0.float().to(dev),
                                    bi.to(dev), cd if dnet else None, dth, ATHR, 3.05, 1.0, times,
                                    return_counters=True, mode="tc")


@pytest.mark.parametrize("pair", list(TC_PAIRS))
def test_tc_trace_matches_fp64_oracle(cuda_dev, pair):
    """Convergence masks match on every insensitive ray, points on kept rays meet ELEM + 2 e_f, and each iteration's update
    count is the oracle's up to the sensitive rays.

    Sensitive rays are marked with the engine's error bounds (ops.TC_EPS_F on f, 1e-3 degrees on the angle).  A ray is
    ill-conditioned, excluded and counted, when the float64 trajectory moves by more than ELEM / 2 with every SDF value
    off by the engine's error measured at the start points (+-, below TC_EPS_F).  At most 5 % may be excluded that way after one or two iterations.  Ten
    iterations amplify an f error on the rays that keep failing the angle test: with this rule the float64 oracle alone
    excludes 4-11 % of 160 rays at an f error of 4e-6-1e-5 (perturbing by TC_EPS_F itself, 20 %), so there the cap
    is 20 %.  A kernel bug moves most updated rays, so either cap still rejects it.  Rays whose trajectory takes a
    gradient within RELU_MARGIN_TC of a translator ReLU kink are excluded and counted as well."""
    from selfreconcode_b200 import ops
    (triple, n) = TC_PAIRS[pair]
    sdf, dnet, st, cd, x0, bi, cam, rays, f0, sdf_fn, def_fn = _trace_setup(triple, cuda_dev, n, odev=cuda_dev)
    eps = (ops.TC_EPS_F, 1e-3)
    # the engine's error on f at the start points
    f_tc = ops.tc_mlp_forward(sdf.fused.truncated_last(1), x0.float())[:, 0].double()
    with torch.no_grad():
        e_f = float((f_tc - sdf_fn(x0).view(-1)).abs().max())
    print("tc trace %s, %d rays: engine's |f| error at the start points %.2e (bound %.0e)" % (pair, n, e_f, eps[0]))
    assert e_f < eps[0]
    # Points: ELEM, plus the measured f error twice over (a Newton step moves a point by about its f error, |grad f| ~ 1;
    # once at the start point, once at the last iterate): the elementwise bar of the fp32 engines does not leave room
    # for the tensor-core engine's error on f, 10 times theirs.
    bar = ELEM + 2 * e_f
    dth = _split_threshold(cam, rays, x0, bi, sdf_fn, def_fn, f0)
    cases = [("split", dth, 1), ("split", dth, 2), ("split", dth, 10), ("all converge", 1e3, 10),
             ("none converge", 0.0, 2), ("none converge", 0.0, 10)]
    rel = lambda a, b: ((a - b).abs() / (b.abs() + b.abs().mean())).amax(1)
    for label, d, times in cases:
        po, co, sens, iters = _oracle_trace(cam, rays, x0, bi, sdf_fn, def_fn, d, times, eps, with_iters=True)
        pt, ct, cnt = _tc_trace(sdf, dnet, st, cd, x0, rays, bi, d, times)
        moved = torch.zeros(n, dtype=torch.bool, device=cuda_dev)
        for pert in (lambda p: sdf_fn(p) + e_f, lambda p: sdf_fn(p) - e_f):
            moved |= rel(_oracle_trace(cam, rays, x0, bi, pert, def_fn, d, times, eps)[0], po) > ELEM / 2
        kinked = ~_kink_free(dnet, cd, cam, rays, x0, bi, sdf_fn, def_fn, d, times, iters) & ~sens
        moved &= ~sens & ~kinked
        keep = ~sens & ~moved & ~kinked
        over = int(((rel(pt.double(), po) > bar) & keep).sum())
        mism = int(((ct != co) & ~sens).sum())
        ns = int(sens.sum())
        ocnt = [int(((iters >= k) & ~sens).sum()) for k in range(1, times + 1)]
        got = cnt[1:times + 1].tolist()
        print("tc trace %s %s times=%d: dthreshold %.3g, %d of %d converged, %d sensitive, %d ill-conditioned, "
              "%d near a ReLU kink, %d mismatches; updates %s (oracle, insensitive: %s); %d kept rays over the bar"
              % (pair, label, times, d, int(co.sum()), n, ns, int(moved.sum()), int(kinked.sum()), mism, got, ocnt,
                 over))
        # ten gradients per ray each risk a kink (8 % of the rays at one): after ten iterations fewer rays are kept
        assert keep.float().mean() > (0.5 if times <= 2 else 0.3)
        assert int(moved.sum()) <= (0.05 if times <= 2 else 0.2) * n, int(moved.sum())
        assert mism == 0
        assert all(o <= c <= o + ns for c, o in zip(got, ocnt)), (got, ocnt, ns)
        if label == "split" and times <= 2:
            assert 0.2 * n <= int(co.sum()) <= 0.8 * n
        if label == "all converge":
            assert bool(co.all()) and sum(got) == 0, "every later launch runs on an empty list"
        if label == "none converge":
            assert not bool(ct.any()) and got == [n] * times
        e = elem_err(pt[keep].cpu().numpy(), po[keep].cpu().numpy())
        print("  %-40s elem %.2e  (bar %.2e)" % ("points", e, bar))
        assert e < bar, ("points", e)


# ---------------------------------------------------------------------------------------------------------------------
# invariances and plumbing of _trace_surface_points_tc
# ---------------------------------------------------------------------------------------------------------------------
P_INV = 2 * WAVE_WARP + 77          # a ragged last tile (77 rows); a second wave of trace_mid and of the row tiles


def _production_setup(dev, n):
    sdf, dnet, st, cd, x0, bi, cam, rays, f0, sdf_fn, def_fn = _trace_setup(("ref_sdf", "translator_ref", True), dev,
                                                                            n, odev=dev)
    return sdf, dnet, st, cd, x0.float(), bi, rays.float(), float(f0.quantile(0.3))


def test_tc_trace_invariance_bitwise(cuda_dev):
    """A row's arithmetic does not depend on its tile or its list position: permutation, the first 17 rays alone and a
    rerun (eager, then through the captured graph) give the same bits."""
    sdf, dnet, st, cd, x0, bi, rays, dth = _production_setup(cuda_dev, P_INV)

    def run(x, r, b):
        p, c, _ = _tc_trace(sdf, dnet, st, cd, x, r, b, dth, 3)
        return p, c
    _invariant(run, (x0, rays, bi), P_INV, "tc trace")


def test_tc_trace_dual_stream_matches_single_stream(cuda_dev, monkeypatch):
    from selfreconcode_b200 import ops
    sdf, dnet, st, cd, x0, bi, rays, dth = _production_setup(cuda_dev, P_INV)
    res = {}
    for dual in (True, False):
        monkeypatch.setattr(ops, "TC_DUAL_STREAM", dual)
        res[dual] = _tc_trace(sdf, dnet, st, cd, x0, rays, bi, dth, 3)
    for a, b in zip(res[True], res[False]):
        assert torch.equal(a, b)
    print("dual / single stream: counters %s" % res[True][2].tolist())


def test_tc_trace_graph_replay_follows_new_contents(cuda_dev, monkeypatch):
    """A captured trace replayed on new pose, latent codes, batch indices, rays and start points equals an eager trace
    of the same contents; so does a configuration evicted (after more than four others) and traced again."""
    from selfreconcode_b200 import ops
    from helpers import golden
    P = 4097
    sdf, dnet, st, cd, x0, bi, rays, dth = _production_setup(cuda_dev, P)
    gd = golden("deform.npz")
    g = torch.Generator().manual_seed(80)
    poses0, trans0 = torch.from_numpy(gd["poses"]).to(cuda_dev), torch.from_numpy(gd["trans"]).to(cuda_dev)
    poses1 = poses0 + (0.05 * torch.randn(poses0.shape, generator=g, dtype=poses0.dtype)).to(cuda_dev)
    trans1 = trans0 + 0.01
    cd1 = cd * 1.3 + 0.05
    bi1 = torch.randint(0, NFRAMES, (P,), generator=g).to(cuda_dev)
    x1 = x0 + (0.01 * torch.randn(P, 3, generator=g)).to(cuda_dev)
    rays1 = torch.nn.functional.normalize(rays + (0.002 * torch.randn(P, 3, generator=g)).to(cuda_dev), dim=1)
    contents = [(poses0, trans0, cd, bi, x0, rays), (poses1, trans1, cd, bi, x0, rays),
                (poses1, trans1, cd1, bi, x0, rays), (poses1, trans1, cd1, bi1, x0, rays),
                (poses0, trans0, cd1, bi1, x1, rays1)]

    def trace(c, times=2):
        st.set_pose(c[0], c[1])
        return _tc_trace(sdf, dnet, st, c[2], c[4], c[5], c[3], dth, times)

    monkeypatch.setattr(ops, "_tc_trace_ctx", {})
    monkeypatch.setattr(ops, "GRAPHS_ENABLED", False)
    eager = [trace(c) for c in contents]
    for k in range(1, len(contents)):
        assert not torch.equal(eager[k][0], eager[k - 1][0]), "each change of contents must change the trace"
    monkeypatch.setattr(ops, "_tc_trace_ctx", {})
    monkeypatch.setattr(ops, "GRAPHS_ENABLED", True)

    def same(k, out, what):
        for a, b in zip(out, eager[k]):
            assert torch.equal(a, b), (what, k)
    same(0, trace(contents[0]), "eager")
    same(0, trace(contents[0]), "capture")
    assert len(ops._tc_trace_ctx) == 1 and next(iter(ops._tc_trace_ctx.values())).graph is not None
    for k, c in enumerate(contents):
        same(k, trace(c), "replay")
    for times in (1, 3, 4, 5, 6):          # five other configurations, each captured: the first one is evicted
        trace(contents[0], times)
        trace(contents[0], times)
    assert len(ops._tc_trace_ctx) == 4
    for k in (3, 4, 2):                    # traced again: eager, capture, replay
        same(k, trace(contents[k]), "after eviction")
    print("graph replay on %d content sets and after eviction: bitwise equal to eager traces" % len(contents))
