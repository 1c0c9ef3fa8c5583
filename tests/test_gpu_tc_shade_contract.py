"""GPU: the tensor-core infer shading (ops.shade_and_render_tc) against float64 restatements at the production networks.

  * its stages on their own fp32 inputs: the SDF's reverse-mode gradient (ops._sdf_grad_tc), sr_tc_embed_backward
    alone, the translator's ch = 4 sweep with latent codes and batch indices, and the renderer's layer chain on the
    engine's own sr_tc_render_embed rows.  Row counts 1, 127, 128, 129 (either side of the 128-row tile), 2433 and one
    past each stage's first grid-stride wave;
  * the whole call against a float64 composite (SDF, translator, LBS, cardinal rays, renderer) in four deformer
    configurations, with deformed normals, and a per-ray colour bound: the renderer's own error plus the first-order
    propagation of the measured input errors through the float64 renderer;
  * invariances, bitwise (permutation, prefix, rerun, dual- against single-stream, the work-buffer cache), the empty
    ray set, and negative controls that each break one piece of the pipeline and must fail a bar.

Error model of the tensor-core layers.  Each dot product of a layer is formed from split-BF16 planes (the dropped
cross terms are <= 2^-16 of each product) and accumulated in fp32 with truncation, K/16 additions per plane pair: at
K <= 512 that is at most 96 truncations of 2^-23, under 2^-16 of the sum of the magnitudes of its terms.  So a layer
adds at most U = 2^-15 of sum |terms| to each pre-activation.  That local error is worst-case; the errors that reach a
unit from the previous layer come through weights of both signs from independent units, so they add in quadrature.
_sigma carries that estimate through the chain (act' scales it; softplus's act'' turns a value error into a tangent
error), and a kernel's output must lie within SIG_K = 3 times it: the estimate of one output is a standard deviation at
most (independent errors each bounded by b have a deviation of at most b / sqrt(3)), and a maximum over ~10^5 outputs
sits near 4-5 deviations, so 3 times the quadrature sum of the bounds covers it.

Every measured maximum is printed beside its bar (pytest -s)."""
import ctypes as C
import math

import pytest
import torch

import ffma_ref as R
from oracle import oracle as O
from test_gpu_ffma_contract import (CONDLEN, ELEM, NFRAMES, _invariant, _lib, _p, _s, _sample, conds,
                                    lbs_pixel, lbs_setup, render_net, sdf_net, sentinel, translator_net, untouched)
from test_gpu_narrow_shade import NORMAL_BAR
from test_gpu_tc_trace_contract import RELU_MARGIN_TC, WAVE_THREAD, WAVE_WARP, _pw

pytestmark = pytest.mark.gpu

U = 2.0 ** -15
SIG_K = 3.0
EPS32 = 2.0 ** -23
FLIP = torch.diag(torch.tensor([-1.0, 1.0, -1.0], dtype=torch.float64))
ROWS = (1, 127, 128, 129, 2433)


# ---------------------------------------------------------------------------------------------------------------------
# the error model and the float64 restatements
# ---------------------------------------------------------------------------------------------------------------------
def _act_d(act, z):
    """act'(z), act''(z) in float64."""
    if act == R.SP:
        s = torch.sigmoid(100.0 * z)
        return s, 100.0 * s * (1.0 - s)
    if act == R.RELU:
        return (z > 0).double(), torch.zeros_like(z)
    if act == R.TANH:
        t = torch.tanh(z)
        return 1.0 - t * t, -2.0 * t * (1.0 - t * t)
    return torch.ones_like(z), torch.zeros_like(z)


def _sigma(layers, inp, d_in, tan=None):
    """Per output: the tensor-core error estimate of the module docstring, for the values and (tan [P, 3, K], the
    input's tangents) for the forward tangents.  A ReLU unit within SIG_K of its estimate of 0 may switch: its value is
    continuous there, so it is carried as if on (a switched unit's output is within its own error)."""
    h, s = inp.double(), U * inp.double().abs()
    x0, s0 = h[:, :d_in], s[:, :d_in]
    t = tan.double() if tan is not None else None
    st = U * t.abs() if t is not None else None
    t0, st0 = (t[..., :d_in], st[..., :d_in]) if t is not None else (None, None)
    for L in layers:
        W = R.effective_weight(L).to(h.device)
        b = L["b"].double().to(h.device) if L.get("b") is not None else torch.zeros(W.shape[0], dtype=torch.float64,
                                                                                 device=h.device)
        if L.get("skip"):
            h, s = torch.cat([h, x0], 1) * R.INV_SQRT2, torch.cat([s, s0], 1) * R.INV_SQRT2
            if t is not None:
                t, st = torch.cat([t, t0], -1) * R.INV_SQRT2, torch.cat([st, st0], -1) * R.INV_SQRT2
        z = h @ W.t() + b
        sz = U * (h.abs() @ W.abs().t() + b.abs()) + ((s * s) @ (W * W).t()).sqrt()
        a1, a2 = _act_d(L["act"], z)
        if L["act"] == R.RELU:
            a1 = (z > -SIG_K * sz).double()
        if t is not None:
            tz = t @ W.t()
            stz = U * (t.abs() @ W.abs().t()) + ((st * st) @ (W * W).t()).sqrt()
            st = a1.unsqueeze(1) * stz + a2.abs().unsqueeze(1) * tz.abs() * sz.unsqueeze(1)
            t = a1.unsqueeze(1) * tz
        h, s = R.activation(L["act"], z), a1 * sz
    return h, s, t, st


def _relu_sigma_margin(layers, inp):
    """Per row: min over the ReLU units of |z| / (SIG_K sigma_z), sigma_z being _sigma's error estimate of z."""
    h, s = inp.double(), U * inp.double().abs()
    m = torch.full((h.shape[0],), math.inf, dtype=torch.float64, device=h.device)
    for L in layers:
        W = R.effective_weight(L).to(h.device)
        b = L["b"].double().to(h.device)
        z = h @ W.t() + b
        sz = U * (h.abs() @ W.abs().t() + b.abs()) + ((s * s) @ (W * W).t()).sqrt()
        if L["act"] == R.RELU:
            m = torch.minimum(m, (z.abs() / (SIG_K * sz)).min(1).values)
        a1 = (z > -SIG_K * sz).double() if L["act"] == R.RELU else _act_d(L["act"], z)[0]
        h, s = R.activation(L["act"], z), a1 * sz
    return m


def _embed_tangent(x, multires, pw):
    """d embed / d x_c for c = 0..2: [P, 3, 3 + 6 multires] in float64."""
    x = x.double()
    P = x.shape[0]
    T = torch.zeros(P, 3, 3 + 6 * multires, dtype=torch.float64, device=x.device)
    for c in range(3):
        T[:, c, c] = 1.0
        for b in range(multires):
            fr = 2.0 ** b
            T[:, c, 3 + 6 * b + c] = pw[b] * fr * torch.cos(fr * x[:, c])
            T[:, c, 6 + 6 * b + c] = -pw[b] * fr * torch.sin(fr * x[:, c])
    return T


def _prod(dev):
    st, lref = lbs_setup(dev)
    rnet, nfeat = render_net("render_ref", dev)
    return dict(sdf=sdf_net("ref_sdf", dev), dnet=translator_net("translator_ref", dev), rnet=rnet, nfeat=nfeat,
                st=st, lref=lref, cd=conds(dev))


def _render_in(rnet, pts, nrm, views, feat):
    """The renderer's input rows in float64, as sr_tc_render_embed lays them out (differentiable in each part)."""
    return torch.cat([pts.double(), R.embed(views, rnet.multires, rnet.pe_w), nrm.double(), feat.double()], 1)


def _composite64(N, pts, rays, bi, with_def, with_lbs, R0=None, sigma_kinks=False):
    """shade_and_render_tc in float64 on fp32 points: normals, grad f, features, offset and d offset / dp, D(p), M, J,
    inv_ok, cardinal rays, deformed normals (camera frame with R0), rgb; and the translator's ReLU margin."""
    dev = pts.device
    P = pts.shape[0]
    sdf, dnet, lref, cd = N["sdf"], N["dnet"] if with_def else None, N["lref"] if with_lbs else None, N["cd"]
    f, g, out = R.sdf(sdf.layers, pts, sdf.multires, sdf.pe_w)
    eye = torch.eye(3, dtype=torch.float64, device=dev).expand(P, 3, 3)
    if dnet is not None:
        off, Joff = R.jacobian(lambda x: R.translator_offset(dnet.layers, x, 6, dnet.pe_w, cd, bi), pts)
        with torch.no_grad():
            _, zs = R.translator_offset(dnet.layers, pts.double(), 6, dnet.pe_w, cd, bi, with_preacts=True)
        margin = R.min_relu_margin(dnet.layers, zs)
        if sigma_kinks:
            # a unit is near its kink when |z| is within SIG_K of _sigma's error estimate of z: expressed on the
            # RELU_MARGIN_TC scale the rest of the file uses
            inp = torch.cat([R.embed(pts, 6, dnet.pe_w), cd.double()[bi]], 1)
            margin = RELU_MARGIN_TC * _relu_sigma_margin(dnet.layers, inp)
    else:
        off, Joff = torch.zeros(P, 3, dtype=torch.float64, device=dev), torch.zeros_like(eye)
        margin = torch.full((P,), math.inf, dtype=torch.float64, device=dev)
    p1 = pts.double() + off
    if lref is not None:
        D, M = R.jacobian(lambda x: O.lbs_forward(lref["ws"], lref["bmin"], lref["bmax"], lref["A"], lref["trans"], x,
                                                  bi), p1)
    else:
        D, M = p1, eye
    J = M @ (eye + Joff)
    Jinv, ok = O.minv3x3(J)
    v = rays.double()
    cr = torch.where(ok.view(-1, 1), (Jinv @ v.unsqueeze(-1)).squeeze(-1), v)
    cr = cr / cr.norm(dim=1, keepdim=True)
    y = torch.where(ok.view(-1, 1), (Jinv.transpose(1, 2) @ g.unsqueeze(-1)).squeeze(-1),
                    (J @ g.unsqueeze(-1)).squeeze(-1))
    dn = y / y.norm(dim=1, keepdim=True)
    if R0 is not None:
        dn = dn @ (FLIP.to(dev) @ R0.double().t()).t()
    n = g / g.norm(dim=1, keepdim=True)
    rnet = N["rnet"]
    rgb = R.mlp(rnet.layers, _render_in(rnet, pts, n, cr, out[:, 1:]), rnet.d_in)
    return dict(n=n, g=g, f=f, feat=out[:, 1:], off=off, Joff=Joff, D=D, M=M, J=J, ok=ok, cr=cr, dn=dn, rgb=rgb,
                margin=margin)


def _ratio(err, bar):
    """The worst err / bar; a non-finite error fails every bar."""
    if not err.numel():
        return 0.0
    r = err / bar
    return float(r.max()) if bool(torch.isfinite(r).all()) else math.inf


# ---------------------------------------------------------------------------------------------------------------------
# (a) ops._sdf_grad_tc at the production SDF
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pe", ["ones", "annealed"])
def test_sdf_grad_matches_fp64(cuda_dev, pe):
    """f within ops.TC_EPS_F; the 256 features within SIG_K times their error estimate; grad f within NORMAL_BAR of
    |grad f| per component and the normals within NORMAL_BAR, now against float64; reverse mode no worse than the same
    engine's forward tangents."""
    from selfreconcode_b200 import ops
    from test_gpu_ffma_contract import Net
    lib = _lib()
    base = sdf_net("ref_sdf", cuda_dev)
    pw = [1.0] * 6 if pe == "ones" else R.annealing_weights(6, 0.6)
    if pe == "annealed":
        assert 0.0 in pw and any(0.0 < w < 1.0 for w in pw)
    net = Net(base.layers, 39, 6, pw, cuda_dev)
    assert [L.n for L in net.desc.layer[:net.desc.n_layers]] == [512] * 3 + [473] + [512] * 4 + [257]
    sizes = ROWS + (WAVE_THREAD // 64 + 3,)               # the embedding's grid wraps at 64-wide rows
    pts = _sample(sizes[-1], 11, -0.8, 0.8).to(cuda_dev)
    f64, g64, out64 = R.sdf(net.layers, pts, 6, pw)
    n64 = g64 / g64.norm(dim=1, keepdim=True)
    _, s_out, _, _ = _sigma(net.layers, R.embed(pts, 6, pw), 39)
    worst = dict(f=0.0, feat=0.0, grad=0.0, normals=0.0)
    print("sdf_grad_tc, PE %s" % pe)
    for P in sizes:
        out, grad, _ = ops._sdf_grad_tc(lib, net.fused, pts[:P].contiguous(), P)
        torch.cuda.synchronize()
        e_f = float((out[:, 0].double() - f64[:P]).abs().max())
        r_feat = _ratio((out[:, 1:].double() - out64[:P, 1:]).abs(), SIG_K * s_out[:P, 1:])
        e_g = float(((grad.double() - g64[:P]).abs() / g64[:P].norm(dim=1, keepdim=True)).max())
        n = torch.nn.functional.normalize(grad, dim=1)
        e_n = float((n.double() - n64[:P]).abs().max())
        print("  P=%-6d |f| err %.2e (bar %.0e)  features %.3f of the bar  grad f %.2e of |grad f|  normals %.2e "
              "(bar %.0e)" % (P, e_f, ops.TC_EPS_F, r_feat, e_g, e_n, NORMAL_BAR))
        for k, v in (("f", e_f / ops.TC_EPS_F), ("feat", r_feat), ("grad", e_g / NORMAL_BAR),
                     ("normals", e_n / NORMAL_BAR)):
            worst[k] = max(worst[k], v)
    assert all(v <= 1.0 for v in worst.values()), worst
    # Reverse mode against the forward tangents of the same engine, at the largest count.  Against float64 the
    # reverse-mode normals are the less accurate of the two (H100: 2.9e-5 against 2.7e-5 with all band weights 1,
    # 1.6e-5 against 0.9e-5 annealed; DESIGN.md section 4), so only the shared bar is asserted here;
    # test_gpu_narrow_shade keeps the comparison against the FFMA engine.
    g4 = ops.tc_mlp_forward(net.fused, pts, ch=4, n_out=1).view(-1, 4)[:, 1:]
    e_fwd = float((torch.nn.functional.normalize(g4, dim=1).double() - n64).abs().max())
    print("  normals: reverse mode %.2e, forward tangents %.2e (bar %.0e)" % (e_n, e_fwd, NORMAL_BAR))
    assert e_fwd < NORMAL_BAR


# ---------------------------------------------------------------------------------------------------------------------
# (b) sr_tc_embed_backward alone
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_gk,ch", [(True, 1), (False, 1), (False, 4)])
def test_embed_backward_matches_fp64(cuda_dev, with_gk, ch):
    """d/dp of sum(gx . embed(p)) (+ gk on the value row; with ch = 4 also the tangent rows' cotangents through
    d embed / dp_j), within 2^-19 of the sum of the magnitudes of its terms (_chain_scale's, with the trigonometric
    factors bounded by 1: sincosf's error is absolute); nothing written past P rows."""
    lib = _lib()
    mr, ld = 6, 64
    pw = R.annealing_weights(6, 0.6)
    assert 0.0 in pw and any(0.0 < w < 1.0 for w in pw)
    print("embed_backward gk=%d ch=%d" % (with_gk, ch))
    for P in ROWS + (WAVE_THREAD + 77,):
        g = torch.Generator().manual_seed(90 + P)
        x = _sample(P, 91 + P, -1.2, 1.2).to(cuda_dev)
        gx = torch.randn(P * ch, ld, generator=g).to(cuda_dev)
        gk = torch.randn(P, ld, generator=g).to(cuda_dev) if with_gk else None
        out = sentinel(P * 3, cuda_dev)
        assert lib.sr_tc_embed_backward(_p(x), P, mr, _pw(pw), ch, _p(gx), ld, _p(gk), ld if with_gk else 0, _p(out),
                                        _s()) == 0
        torch.cuda.synchronize()
        assert untouched(out, P * 3), P
        got = out[:P * 3].view(P, 3).double()
        pe = 3 + 6 * mr
        G = gx.view(P, ch, ld)[:, :, :pe].double()
        cot = G[:, 0] + (gk[:, :pe].double() if gk is not None else 0.0)
        xd = x.double().requires_grad_(True)
        obj = (R.embed(xd, mr, pw) * cot).sum()
        wf = torch.tensor([pw[b] * 2.0 ** b for b in range(mr)], dtype=torch.float64, device=cuda_dev)
        scale = cot[:, :3].abs() + sum(wf[b] * (cot[:, 3 + 6 * b:6 + 6 * b].abs() + cot[:, 6 + 6 * b:9 + 6 * b].abs())
                                       for b in range(mr))
        if ch == 4:
            T = _embed_tangent(xd, mr, pw)
            obj = obj + (T * G[:, 1:]).sum()
            for j in range(3):
                scale[:, j] += G[:, 1 + j, j].abs() + sum(wf[b] * 2.0 ** b * (G[:, 1 + j, 3 + 6 * b + j].abs() +
                                                                               G[:, 1 + j, 6 + 6 * b + j].abs())
                                                          for b in range(mr))
        (ref,) = torch.autograd.grad(obj, xd)
        r = _ratio((got - ref).abs(), 2.0 ** -19 * scale)
        print("  P=%-7d max |err| %.2e  (%.3f of the bar)" % (P, float((got - ref).abs().max()), r))
        assert r <= 1.0, P


# ---------------------------------------------------------------------------------------------------------------------
# (c) the translator's ch = 4 sweep
# ---------------------------------------------------------------------------------------------------------------------
def test_translator_tangent_sweep_matches_fp64(cuda_dev):
    """Row 4p = offset, rows 4p+1+c = d offset / dp_c, within SIG_K times _sigma's estimate for values and tangents.
    Points with a ReLU unit within RELU_MARGIN_TC of its kink switch d offset / dp: excluded, counted, capped."""
    from selfreconcode_b200 import ops
    dnet, cd = translator_net("translator_ref", cuda_dev), conds(cuda_dev)
    sizes = ROWS + (WAVE_THREAD // (4 * 192) + 1,)          # the ch = 4 embedding's grid wraps at 4 rows of 192
    Pm = max(sizes)
    pts = _sample(Pm, 120, -0.8, 0.8).to(cuda_dev)
    bi = torch.randint(0, NFRAMES, (Pm,), generator=torch.Generator().manual_seed(121)).to(cuda_dev)
    off64, J64 = R.jacobian(lambda x: R.translator_offset(dnet.layers, x, 6, dnet.pe_w, cd, bi), pts)
    inp = torch.cat([R.embed(pts, 6, dnet.pe_w), cd.double()[bi]], 1)
    tan = torch.cat([_embed_tangent(pts, 6, dnet.pe_w), torch.zeros(Pm, 3, CONDLEN, dtype=torch.float64,
                                                                     device=cuda_dev)], 2)
    _, s_off, _, s_t = _sigma(dnet.layers, inp, inp.shape[1], tan)
    with torch.no_grad():
        _, zs = R.translator_offset(dnet.layers, pts.double(), 6, dnet.pe_w, cd, bi, with_preacts=True)
    keep = R.min_relu_margin(dnet.layers, zs) >= RELU_MARGIN_TC
    print("translator ch=4: %d of %d points within %.0e of a ReLU kink, excluded" % (int((~keep).sum()), Pm,
                                                                                    RELU_MARGIN_TC))
    assert (~keep).float().mean() < 0.15
    for P in sizes:
        o4 = ops.tc_mlp_forward(dnet.fused, pts[:P], ch=4, conds=cd, batch_inds=bi[:P]).view(P, 4, 3).double()
        k = keep[:P]
        r_off = _ratio((o4[:, 0] - off64[:P]).abs()[k], SIG_K * s_off[:P][k])
        # tangent row c holds d offset_i / dp_c = J64[:, i, c]; s_t [P, c, i]
        r_t = _ratio((o4[:, 1:] - J64[:P].transpose(1, 2)).abs()[k], SIG_K * s_t[:P][k])
        e_t = float((o4[:, 1:] - J64[:P].transpose(1, 2)).abs()[k].max()) if int(k.sum()) else 0.0
        print("  P=%-5d offset %.3f of the bar, tangents %.3f of the bar (max |err| %.2e)" % (P, r_off, r_t, e_t))
        assert r_off <= 1.0 and r_t <= 1.0, P


# ---------------------------------------------------------------------------------------------------------------------
# (d) the renderer's layer chain on the engine's own input rows
# ---------------------------------------------------------------------------------------------------------------------
def _render_tc(lib, rnet, pts, nrm, views, feat, pw=None, col0=1, feat_ld=None):
    """sr_tc_render_embed + the renderer's tensor-core chain, as shade_and_render_tc runs them; returns (rows, rgb)."""
    from selfreconcode_b200 import ops
    P = pts.shape[0]
    rd = rnet.fused.desc
    ld = (rd.d_in + 31) // 32 * 32
    emb = torch.empty(P, ld, device=pts.device)
    pwc = _pw(rnet.pe_w if pw is None else pw)
    assert lib.sr_tc_render_embed(P, _p(pts), _p(views), _p(nrm), _p(feat), feat.shape[1], col0, 256, 1, rd.multires,
                                  pwc, _p(emb), ld, _s()) == 0
    buf = sentinel(P * 3, pts.device)
    ops._tc_mlp(lib, ops.tc_net(rnet.fused), emb, 1, buf[:P * 3].view(P, 3))
    torch.cuda.synchronize()
    assert untouched(buf, P * 3)
    return emb, buf[:P * 3].view(P, 3)


def test_render_chain_matches_fp64(cuda_dev):
    """rgb from the engine's own fp32 render_embed rows within SIG_K times _sigma's estimate on those rows: the
    renderer's GEMM error alone.  No row is excluded: a ReLU unit within reach of its kink is carried by _sigma as if on
    (the values are continuous there, so a switched unit's output is within its own error)."""
    from test_gpu_ffma_contract import render_inputs
    lib = _lib()
    rnet, nfeat = render_net("render_ref", cuda_dev)
    sizes = ROWS + (WAVE_THREAD // 320 + 3,)               # render_embed's grid wraps at 320-wide rows
    Pm = max(sizes)
    pts, nrm, views, feat = render_inputs(Pm, nfeat, cuda_dev, 130)
    feat = torch.cat([torch.zeros(Pm, 1, device=cuda_dev), feat], 1)        # the SDF's output row: f, then features
    print("render chain")
    for P in sizes:
        emb, rgb = _render_tc(lib, rnet, pts[:P], nrm[:P], views[:P], feat[:P].contiguous())
        rows = emb[:, :rnet.d_in].double()
        rgb64, zs = R.mlp(rnet.layers, rows, rnet.d_in, with_preacts=True)
        _, s, _, _ = _sigma(rnet.layers, rows, rnet.d_in)
        r = _ratio((rgb.double() - rgb64).abs(), SIG_K * s)
        print("  P=%-6d max |err| %.2e  (%.3f of the bar)" % (P, float((rgb.double() - rgb64).abs().max()), r))
        assert r <= 1.0, P


# ---------------------------------------------------------------------------------------------------------------------
# 2. shade_and_render_tc end to end
# ---------------------------------------------------------------------------------------------------------------------
CONFIGS = {"translator_lbs": (True, True), "translator": (True, False), "lbs": (False, True), "identity": (False, False)}


def _shade_points(N, with_def, with_lbs, dev, n=WAVE_WARP + 77 - 129, n_out=129):
    """Tensor-core traced points (converged and not: the bench shades every ray's point) and points outside the
    skinning box."""
    from test_gpu_ffma_contract import _trace_setup
    from test_gpu_tc_trace_contract import _tc_trace
    triple = ("ref_sdf", "translator_ref" if with_def else None, with_lbs)
    sdf, dnet, st, cd, x0, bi, cam, rays, f0, _, _ = _trace_setup(triple, dev, n, odev=dev)
    pt, conv, _ = _tc_trace(sdf, dnet, st, cd, x0, rays, bi, float(f0.quantile(0.3)), 10)
    lo, hi = N["lref"]["bmin"].float(), N["lref"]["bmax"].float()
    g = torch.Generator().manual_seed(140)
    sgn = torch.where(torch.rand(n_out, 3, generator=g) < 0.5, -1.0, 1.0).to(dev)
    outside = (lo + hi) / 2 + sgn * (hi - lo) * (0.55 + 0.2 * torch.rand(n_out, 3, generator=g).to(dev))
    ro = torch.nn.functional.normalize(torch.randn(n_out, 3, generator=g), dim=1).to(dev)
    bo = torch.randint(0, NFRAMES, (n_out,), generator=g).to(dev)
    return (torch.cat([pt, outside]).contiguous(), torch.cat([rays.float(), ro]).contiguous(), torch.cat([bi, bo]),
            int(conv.sum()))


def _rotation(seed):
    q = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(seed), dtype=torch.float64))[0]
    return (q * torch.sign(torch.linalg.det(q))).float()


def _engine(N, with_def, with_lbs, pts, rays, bi, R0=None, mut=None):
    """shade_and_render_tc restated launch by launch (bitwise the same, asserted below), with the negative controls'
    mutations: 'col0' features from column 0, 'anneal' the view encoding's weights ignored, 'nrm0' the renderer's
    normal columns zeroed, 'noskip' the skip part of grad f dropped, 'jT' the translator's tangent block transposed,
    'noM' M = I with LBS on (LBS dropped from the pointwise pass), 'R0T' cam_R0 transposed, 'Jsing' the translator's
    tangent block set to -I (J = 0: every point takes the singular fallback)."""
    from selfreconcode_b200 import ops
    lib = _lib()
    P = pts.shape[0]
    sdf, dnet, st, rnet = N["sdf"], N["dnet"] if with_def else None, N["st"] if with_lbs else None, N["rnet"]
    out, grad, g_out = (t.clone() for t in ops._sdf_grad_tc(lib, sdf.fused, pts, P))
    if mut == "noskip":
        grad = torch.empty(P, 3, device=pts.device)
        assert lib.sr_tc_embed_backward(_p(pts), P, 6, _pw(sdf.pe_w), 1, _p(g_out), g_out.shape[1], None, 0, _p(grad),
                                        _s()) == 0
    o4 = ops.tc_mlp_forward(dnet.fused, pts, ch=4, conds=N["cd"], batch_inds=bi) if dnet is not None else None
    o4_in = o4                     # the stage's output (its measured error feeds the bars) and what shading reads
    if mut == "jT" and o4 is not None:
        b = o4.view(P, 4, 3).clone()
        b[:, 1:] = b[:, 1:].transpose(1, 2)
        o4_in = b.view(P * 4, 3).contiguous()
    if mut == "Jsing" and o4 is not None:
        b = o4.view(P, 4, 3).clone()
        b[:, 1:] = -torch.eye(3, device=pts.device)
        o4_in = b.view(P * 4, 3).contiguous()
    lbs = None if mut == "noM" else st
    nrm, cr, dp = (torch.empty(P, 3, device=pts.device) for _ in range(3))
    ok = torch.empty(P, dtype=torch.bool, device=pts.device)
    dn = torch.empty(P, 3, device=pts.device)
    Rm = R0.t() if (mut == "R0T" and R0 is not None) else R0
    r0 = (C.c_float * 9)(*Rm.reshape(9).tolist()) if Rm is not None else None
    assert lib.sr_tc_shade_point_deformed(P, _p(pts), _p(rays), _p(bi), _p(grad), _p(o4_in), C.byref(lbs.params) if lbs
                                          else None, _p(nrm), _p(cr), _p(dp), _p(ok), _p(dn), r0, _s()) == 0
    nin = torch.zeros_like(nrm) if mut == "nrm0" else nrm
    _, rgb = _render_tc(lib, rnet, pts, nin, cr, out, pw=[1.0] * 4 if mut == "anneal" else None,
                        col0=0 if mut == "col0" else 1)
    return dict(n=nrm, cr=cr, rgb=rgb, D=dp, ok=ok, dn=dn, grad=grad, feat=out[:, 1:], o4=o4)


def _bars(N, E, ref, with_def, with_lbs, pts, R0=None, drop=None):
    """Per bar: the worst ratio of error to bar over the kept points, and the exclusion counts.  `drop` (0: normals,
    1: cardinal rays, 2: features) leaves that input's term out of the colour bound: a negative control of the bound."""
    P = pts.shape[0]
    dev = pts.device
    o4 = E["o4"].view(P, 4, 3).double() if E["o4"] is not None else None
    d_off = (o4[:, 0] - ref["off"]).norm(dim=1) if o4 is not None else torch.zeros(P, dtype=torch.float64, device=dev)
    d_joff = (o4[:, 1:].transpose(1, 2) - ref["Joff"]).flatten(1).norm(dim=1) if o4 is not None else torch.zeros_like(
        d_off)
    Mn = torch.linalg.matrix_norm(ref["M"], ord=2)
    # J error per row: M times the measured error of d offset / dp, plus M's fp32 rounding (2^-18 of |J|)
    d_J = Mn * d_joff + 2.0 ** -18 * torch.linalg.matrix_norm(ref["J"], ord=2)
    sv = torch.linalg.svdvals(ref["J"])
    inv_n = 1.0 / sv[:, 2]
    kappa = sv[:, 0] / sv[:, 2]
    # exclusions: ReLU kinks of the translator, p + offset within the measured offset error of a voxel face, |det J|
    # within its error of the 1e-4 threshold
    kink = ref["margin"] < RELU_MARGIN_TC
    face = torch.zeros(P, dtype=torch.bool, device=dev)
    if with_lbs:
        lref = N["lref"]
        x, size = lbs_pixel(lref, pts.double() + ref["off"])
        world = (lref["bmax"] - lref["bmin"]) / size
        reach = (float(d_off.max()) + 1e-6)
        face = (((x - x.round()).abs() * world < reach) & (x > -1.0) & (x < size)).any(1)
    det = torch.linalg.det(ref["J"])
    d_det = 3.0 * sv[:, 0] ** 2 * d_J
    near_det = (det.abs() - 1e-4).abs() < d_det
    keep = ~kink & ~face & ~near_det
    ok64 = ref["ok"]
    res = {}
    res["inv_ok"] = float(((E["ok"] != ok64) & keep).sum())          # must be 0
    res["normals"] = _ratio((E["n"].double() - ref["n"]).abs().max(1).values[keep], torch.full_like(d_off[keep],
                                                                                                  NORMAL_BAR))
    res["D"] = _ratio((E["D"].double() - ref["D"]).norm(dim=1)[keep],
                      (Mn * d_off + 2.0 ** -19 * (1.0 + ref["D"].norm(dim=1)))[keep])
    # cardinal rays: normalize(J^-1 v).  J + dJ changes J^-1 v by at most |J^-1| dJ relative to it, which moves the
    # unit vector by at most twice that; the kernel's own rounding is test_entry_point_vs_float64's 32 eps kappa amp,
    # with amp = |J^-1| |v| / |J^-1 v| <= kappa
    rnd = 32 * EPS32 * (kappa * kappa + 1.0)
    bar_cr = torch.where(ok64, 2.0 * inv_n * d_J + rnd, torch.full_like(inv_n, 32 * EPS32))
    res["cardinal rays"] = _ratio((E["cr"].double() - ref["cr"]).norm(dim=1)[keep & ok64], bar_cr[keep & ok64])
    g = ref["g"]
    d_g = (E["grad"].double() - g).norm(dim=1)
    y = (ref["J"].inverse().transpose(1, 2) @ g.unsqueeze(-1)).squeeze(-1)
    bar_dn = 2.0 * (inv_n * d_J + inv_n * d_g / y.norm(dim=1)) + rnd
    res["deformed normals"] = _ratio((E["dn"].double() - ref["dn"]).norm(dim=1)[keep & ok64], bar_dn[keep & ok64])
    # rgb, per ray and channel: the renderer's own error on the ray's engine rows (itself within stage (d)'s bar) plus
    # the first-order propagation of the measured input errors through the float64 renderer.  The first-order term is
    # exact up to second order only where both rows switch the same ReLU units: a ray whose float64 renderer switches a
    # unit between its engine rows and its float64 rows is excluded and counted (the renderer's ReLU margin is the
    # pre-activation change the measured input error causes).
    rnet = N["rnet"]
    ins = [ref["n"].detach().clone().requires_grad_(True), ref["cr"].detach().clone().requires_grad_(True),
           ref["feat"].detach().clone().requires_grad_(True)]
    rgb64 = R.mlp(rnet.layers, _render_in(rnet, pts, ins[0], ins[1], ins[2]), rnet.d_in)
    dins = [E["n"].double() - ref["n"], E["cr"].double() - ref["cr"], E["feat"].double() - ref["feat"]]
    prop = torch.zeros(P, 3, dtype=torch.float64, device=dev)
    for c in range(3):
        gr = torch.autograd.grad(rgb64[:, c].sum(), ins, retain_graph=c < 2)
        for i, (gi, di) in enumerate(zip(gr, dins)):
            if i != drop:
                prop[:, c] += (gi.abs() * di.abs()).sum(1)
    with torch.no_grad():
        rows = _render_in(rnet, pts, E["n"], E["cr"], E["feat"])
        r_rows, z_tc = R.mlp(rnet.layers, rows, rnet.d_in, with_preacts=True)
        _, z64 = R.mlp(rnet.layers, _render_in(rnet, pts, ref["n"], ref["cr"], ref["feat"]), rnet.d_in,
                       with_preacts=True)
    rkink = torch.zeros(P, dtype=torch.bool, device=dev)
    for L, za, zb in zip(rnet.layers, z_tc, z64):
        if L["act"] == R.RELU:
            rkink |= ((za > 0) != (zb > 0)).any(1)
    _, s_r, _, _ = _sigma(rnet.layers, rows, rnet.d_in)
    e_own = (E["rgb"].double() - r_rows).abs()
    e_rgb = (E["rgb"].double() - ref["rgb"]).abs()
    kr = keep & ~rkink
    res["rgb"] = max(_ratio(e_rgb[kr], (e_own + prop * (1.0 + 1e-3) + 1e-12)[kr]), _ratio(e_own[kr], SIG_K * s_r[kr]))
    top = lambda t: float(t[kr].max()) if int(kr.sum()) else 0.0          # noqa: E731
    res["_rgb_max"], res["_rgb_own"], res["_rgb_prop"] = top(e_rgb), top(e_own), top(prop)
    res["_rgb_elem"] = float((e_rgb > ELEM * (ref["rgb"].abs() + ref["rgb"].abs().mean())).any(1)[kr].float().mean()) \
        if int(kr.sum()) else 0.0
    res["_excl"] = (int(kink.sum()), int((face & ~kink).sum()), int((near_det & ~kink & ~face).sum()),
                    int((rkink & keep).sum()))
    res["_keep"] = kr
    return res


BAR_NAMES = ("inv_ok", "normals", "D", "cardinal rays", "deformed normals", "rgb")


def _print_bars(head, res):
    kink, face, det, rkink = res["_excl"]
    print("%s; excluded: %d translator ReLU kink, %d voxel face, %d |det J| at 1e-4, %d renderer ReLU switch"
          % (head, kink, face, det, rkink))
    for k in BAR_NAMES:
        print("  %-20s %s" % (k, ("%d mismatches" % res[k]) if k == "inv_ok" else "%.3f of the bar" % res[k]))
    print("  rgb max |err| %.2e (renderer's own %.2e, propagated inputs up to %.2e); %.2f %% of the kept rays above "
          "ELEM" % (res["_rgb_max"], res["_rgb_own"], res["_rgb_prop"], 100 * res["_rgb_elem"]))


def _passes(res):
    return res["inv_ok"] == 0 and all(res[k] <= 1.0 for k in BAR_NAMES[1:])


@pytest.mark.parametrize("config", list(CONFIGS))
def test_shade_and_render_tc_matches_fp64_composite(cuda_dev, config):
    """Every kept point within its per-row bound; inv_ok equal to float64's; the deformed-normal call's shared outputs
    bit-identical to the plain call's; the fp32 FFMA engine on the same points within the plain ELEM bar (the positive
    control of the float64 composite)."""
    from selfreconcode_b200 import ops
    from helpers import elem_err
    with_def, with_lbs = CONFIGS[config]
    N = _prod(cuda_dev)
    pts, rays, bi, nconv = _shade_points(N, with_def, with_lbs, cuda_dev)
    P = pts.shape[0]
    R0 = _rotation(5).to(cuda_dev)
    dnet, st = (N["dnet"].fused if with_def else None), (N["st"] if with_lbs else None)
    args = (N["sdf"].fused, dnet, st, N["rnet"].fused, pts, rays, bi, N["cd"])
    plain = ops.shade_and_render_tc(*args)
    dfn = ops.shade_and_render_tc(*args, deformed_normals=True)
    dfr = ops.shade_and_render_tc(*args, deformed_normals=True, cam_R0=R0)
    for a, b, c in zip(plain, dfn[:5], dfr[:5]):
        assert torch.equal(a, b) and torch.equal(a, c)
    E = _engine(N, with_def, with_lbs, pts, rays, bi, R0)
    for a, k in zip(dfr, ("n", "cr", "rgb", "D", "ok", "dn")):
        assert torch.equal(a, E[k]), ("the launch-by-launch restatement", k)
    ref = _composite64(N, pts, rays, bi, with_def, with_lbs, R0)
    res = _bars(N, E, ref, with_def, with_lbs, pts, R0)
    _print_bars("shade %s: %d points (%d traced converged, 129 outside the skinning box)" % (config, P, nconv), res)
    assert sum(res["_excl"][:3]) <= 0.15 * P and res["_excl"][3] <= 0.05 * P
    assert _passes(res), res
    assert res["_rgb_elem"] == 0.0
    # the colour error explained by each input: float64 normals, features, cardinal rays substituted one at a time
    lib = _lib()
    keep = res["_keep"]
    e0 = float((E["rgb"].double() - ref["rgb"]).abs()[keep].max())
    parts = {}
    for name, sub in (("normals", dict(nrm=ref["n"])), ("features", dict(feat=ref["feat"])),
                      ("cardinal rays", dict(views=ref["cr"]))):
        nrm, views = sub.get("nrm", E["n"]).float().contiguous(), sub.get("views", E["cr"]).float().contiguous()
        ft = torch.cat([torch.zeros(P, 1, device=cuda_dev), sub.get("feat", E["feat"]).float()], 1).contiguous()
        _, rgb_s = _render_tc(lib, N["rnet"], pts, nrm, views, ft)
        parts[name] = float((rgb_s.double() - ref["rgb"]).abs()[keep].max())
    print("  rgb max |err| %.2e; with float64 %s" % (e0, ", ".join("%s %.2e" % kv for kv in parts.items())))
    if with_lbs and not with_def:
        return                     # sr_shade_geometry takes LBS only behind a translator
    # the FFMA engine on the same points
    n2, cr2, ft2, _, _ = ops.shade_geometry(N["sdf"].fused, dnet, st, pts, rays, bi, N["cd"], nfeat=256)
    rgb2 = ops.render_forward(N["rnet"].fused, pts, n2, cr2, ft2)
    e32 = elem_err(rgb2[keep].cpu().numpy(), ref["rgb"][keep].cpu().numpy())
    print("  fp32 FFMA engine rgb: elem %.2e (bar %.0e)" % (e32, ELEM))
    assert e32 < ELEM


# each control and the bars it must fail; together they cover every bar
CONTROLS = {"col0": {"rgb"}, "anneal": {"rgb"}, "nrm0": {"rgb"}, "noskip": {"normals"},
            "jT": {"cardinal rays", "deformed normals"}, "noM": {"D", "cardinal rays", "deformed normals"},
            "R0T": {"deformed normals"}, "Jsing": {"inv_ok", "cardinal rays", "deformed normals"}}


def test_negative_controls_cover_every_bar():
    assert set().union(*CONTROLS.values()) == set(BAR_NAMES)


@pytest.mark.parametrize("mut", list(CONTROLS))
def test_negative_controls_fail_their_bars(cuda_dev, mut):
    """Each broken pipeline fails the bars listed for it in CONTROLS.  The colour bound is fed with the measured input
    errors, so a wrong gradient (noskip) shows in the normals bar and not in the colours' propagation check."""
    N = _prod(cuda_dev)
    pts, rays, bi, _ = _shade_points(N, True, True, cuda_dev)
    R0 = _rotation(5).to(cuda_dev)
    ref = _composite64(N, pts, rays, bi, True, True, R0)
    E = _engine(N, True, True, pts, rays, bi, R0, mut=mut)
    res = _bars(N, E, ref, True, True, pts, R0)
    failed = {k for k in BAR_NAMES if (res[k] > 0 if k == "inv_ok" else res[k] > 1.0)}
    print("control %s: %s" % (mut, ", ".join("%s %.3g" % (k, res[k]) for k in BAR_NAMES)))
    assert CONTROLS[mut] <= failed, (mut, failed)


# ---------------------------------------------------------------------------------------------------------------------
# 4. invariances and plumbing
# ---------------------------------------------------------------------------------------------------------------------
P_INV = 2 * WAVE_WARP + 77          # a ragged last row tile; a second wave of the warp-per-point shading stage


def _inv_inputs(N, dev, P):
    g = torch.Generator().manual_seed(150)
    pts = _sample(P, 151, -0.7, 0.7).to(dev)
    rays = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=1).to(dev)
    bi = torch.randint(0, NFRAMES, (P,), generator=g).to(dev)
    return pts, rays, bi


def _call(N, R0=None):
    from selfreconcode_b200 import ops

    def run(p, r, b):
        return ops.shade_and_render_tc(N["sdf"].fused, N["dnet"].fused, N["st"], N["rnet"].fused, p, r, b, N["cd"],
                                       deformed_normals=True, cam_R0=R0)
    return run


def test_shade_invariance_bitwise(cuda_dev):
    N = _prod(cuda_dev)
    _invariant(_call(N, _rotation(6).to(cuda_dev)), _inv_inputs(N, cuda_dev, P_INV), P_INV, "tc shade")


def test_shade_dual_stream_matches_single_stream(cuda_dev, monkeypatch):
    from selfreconcode_b200 import ops
    N = _prod(cuda_dev)
    args = _inv_inputs(N, cuda_dev, P_INV)
    res = {}
    for dual in (True, False):
        monkeypatch.setattr(ops, "TC_DUAL_STREAM", dual)
        res[dual] = _call(N)(*args)
    for a, b in zip(res[True], res[False]):
        assert torch.equal(a, b)


def test_shade_buffer_cache_matches_fresh(cuda_dev, monkeypatch):
    """P, then 40 P (the cache grows), then P again; two SDFs of the same layer shapes alternated: every call equals the
    same call on an empty cache."""
    from selfreconcode_b200 import ops
    from test_gpu_ffma_contract import Net
    N = _prod(cuda_dev)
    layers2 = [dict(L, b=L["b"] * 1.01 + 1e-3) for L in N["sdf"].layers]
    N2 = dict(N, sdf=Net(layers2, 39, 6, N["sdf"].pe_w, cuda_dev))
    P = 2433
    pts, rays, bi = _inv_inputs(N, cuda_dev, 40 * P)
    cases = [(N, P), (N, 40 * P), (N, P), (N2, P), (N, P), (N2, 40 * P), (N, P)]
    monkeypatch.setattr(ops, "_tc_shade_bufs", {})
    cached = [_call(n)(pts[:p], rays[:p], bi[:p]) for n, p in cases]
    assert len(ops._tc_shade_bufs) == 1
    for (n, p), got in zip(cases, cached):
        monkeypatch.setattr(ops, "_tc_shade_bufs", {})
        fresh = _call(n)(pts[:p], rays[:p], bi[:p])
        for a, b in zip(got, fresh):
            assert torch.equal(a, b), p
    assert not torch.equal(cached[0][2], cached[3][2]), "the two SDFs must shade differently"


def test_shade_empty_ray_set(cuda_dev):
    """An empty ray set (trace_surface_points returns one) gives empty outputs of the right shapes, no launch."""
    from selfreconcode_b200 import ops
    N = _prod(cuda_dev)
    e = torch.empty(0, 3, device=cuda_dev)
    b = torch.empty(0, dtype=torch.int64, device=cuda_dev)
    for dn in (False, True):
        out = ops.shade_and_render_tc(N["sdf"].fused, N["dnet"].fused, N["st"], N["rnet"].fused, e, e, b, N["cd"],
                                      deformed_normals=dn)
        assert len(out) == (6 if dn else 5)
        shapes = [tuple(t.shape) for t in out]
        assert shapes == [(0, 3), (0, 3), (0, 3), (0, 3), (0,)] + ([(0, 3)] if dn else [])
        assert out[4].dtype == torch.bool and all(t.device == e.device for t in out)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the benchmark's scene (BASELINE config[1], 50 333 rays)
# ---------------------------------------------------------------------------------------------------------------------
def _bench_nets(sc, dev):
    """The scene's networks as _engine and _composite64 take them: fused nets for the engine, layer lists, the
    skinning volume and the bone transforms in float64 for the composite."""
    from types import SimpleNamespace as NS
    import bench
    from helpers import plain_params, sdf_params, wn_params
    from selfreconcode_b200 import synth
    tr, sk = sc["comp"].defs
    ones6 = [1.0] * 6
    full = sc["sdf"].fused()
    full.set_pe_weights(ones6)
    sp = sdf_params(sc["sdf"])
    sdf_layers = [dict(v=v, g=g.view(-1), b=b, act=R.SP if l < len(sp) - 1 else R.NONE, skip=l == 4)
                  for l, (v, g, b) in enumerate(sp)]
    tp = plain_params(tr)
    tr_layers = [dict(v=w, g=None, b=b, act=R.RELU if l < len(tp) - 1 else R.NONE, skip=False)
                 for l, (w, b) in enumerate(tp)]
    rp = wn_params(sc["rn"])
    r_layers = [dict(v=v, g=g.view(-1), b=b, act=R.RELU if l < len(rp) - 1 else R.TANH, skip=False)
                for l, (v, g, b) in enumerate(rp)]
    poses, trans = sc["conds"][1]
    A, _ = O.bone_transforms(poses.detach().double().cpu(), sk.Js.detach().double().cpu(), synth.SMPL_PARENTS,
                             sk.init_pose.detach().double().cpu())
    lref = dict(ws=sk.ws.detach().double(), bmin=sk.b_min.detach().view(3).double(),
                bmax=sk.b_max.detach().view(3).double(), A=A.to(dev), trans=trans.detach().double())
    st = sk.lbs_state()
    st.set_pose(poses, trans)
    rf = sc["rn"].fused(bench.RATIO)
    return dict(sdf=NS(fused=full, layers=sdf_layers, multires=6, pe_w=ones6, d_in=39),
                dnet=NS(fused=tr.fused(bench.RATIO), layers=tr_layers, pe_w=ones6),
                rnet=NS(fused=rf, layers=r_layers, multires=4, pe_w=[1.0] * 4, d_in=rf.desc.d_in),
                st=st, lref=lref, cd=sc["conds"][0].detach())


def _elem_rows(err, ref):
    return (err > ELEM * (ref.abs() + ref.abs().mean())).any(1)


def test_bench_scene_colours_vs_fp64(cuda_dev):
    """bench.ray_part's colours at the points the engine traced, against the float64 composite at those points (every
    kept ray within its per-ray bound) and at the float64 oracle's own points (the comparison bench.parity_report
    makes, with the oracle's decision-sensitive rays set aside).  The gap is split into the shading error at the same
    points and the colour change between the two traced points; each input's share of the shading error is shown by
    substituting its float64 value into the tensor-core renderer."""
    import bench
    sc = bench.build_scene(cuda_dev, frame_seed=0)
    Rr = sc["rays"]
    rays, init, bi = (Rr[k].to(cuda_dev) for k in ("rays", "init_pts", "batch_inds"))
    P = rays.shape[0]
    assert P == 50333
    pts, conv, rgb = bench.ray_part(sc, rays, init, bi)
    N = _bench_nets(sc, cuda_dev)
    rays, bi = rays.float().contiguous(), bi.to(torch.int64)
    E = _engine(N, True, True, pts.contiguous(), rays, bi)
    assert torch.equal(E["rgb"], rgb), "the launch-by-launch restatement reproduces the bench's colours"
    # the scene's translator starts from a near-zero output layer: its units sit far closer to 0 than the production
    # network's, so a kink is judged against _sigma's estimate of each pre-activation's error
    ref = _composite64(N, pts, rays, bi, True, True, sigma_kinks=True)
    res = _bars(N, E, ref, True, True, pts)
    _print_bars("bench scene, the engine's points: %d rays" % P, res)
    # most of the scene's rays have a translator unit within its error of 0 (its pre-activations cluster there), so
    # only the ray count left is capped: the per-ray bound holds on every ray away from a kink
    assert int(res["_keep"].sum()) >= 2000 and res["_excl"][3] <= 0.05 * P
    assert _passes(res), res
    # the float64 oracle's trace of the same rays
    lref, sl, dl, cd = N["lref"], N["sdf"].layers, N["dnet"].layers, N["cd"]

    def sdf_fn(p):
        return R.mlp(sl, R.embed(p, 6, [1.0] * 6), 39)[:, :1]

    def def_fn(p, b):
        p1 = p + R.translator_offset(dl, p, 6, [1.0] * 6, cd, b)
        return O.lbs_forward(lref["ws"], lref["bmin"], lref["bmax"], lref["A"], lref["trans"], p1, b)
    sens = dict(eps_f=4e-5, eps_a=1e-3)          # the tensor-core engine's error bounds, as bench.py marks them
    cam = torch.as_tensor(sc["cam"]["cam_pos"]).double().view(3).to(cuda_dev)
    po, co, _ = O.optimize_surface_ps(cam, rays.double(), init.double(), bi, sdf_fn, def_fn, 5e-5, sc["ang"], 3.05,
                                      1.0, 10, sensitivity=sens)
    ins = ~sens["sensitive"].to(cuda_dev)
    ref_o = _composite64(N, po, rays, bi, True, True, sigma_kinks=True)
    tc, r64, r64o = E["rgb"].double(), ref["rgb"], ref_o["rgb"]
    over_all = _elem_rows((tc - r64o).abs(), r64o) & ins
    over_shade = _elem_rows((tc - r64).abs(), r64) & ins
    over_trace = _elem_rows((r64 - r64o).abs(), r64o) & ins
    n_ins = int(ins.sum())
    print("  vs the float64 oracle's points, %d insensitive rays (%d mask mismatches): max |drgb| %.2e, %.2f %% above "
          "ELEM" % (n_ins, int(((conv != co) & ins).sum()), float((tc - r64o).abs()[ins].max()),
                    100 * int(over_all.sum()) / n_ins))
    print("    shading (engine vs float64 at the engine's points): max %.2e, %.2f %% above ELEM"
          % (float((tc - r64).abs()[ins].max()), 100 * int(over_shade.sum()) / n_ins))
    print("    tracing (float64 colours at the two points): max %.2e, %.2f %% above ELEM; points max |dp| %.2e"
          % (float((r64 - r64o).abs()[ins].max()), 100 * int(over_trace.sum()) / n_ins,
             float((pts.double() - po).abs()[ins].max())))
    keep = res["_keep"]
    lib = _lib()
    for name, sub in (("normals", dict(nrm=ref["n"])), ("features", dict(feat=ref["feat"])),
                      ("cardinal rays", dict(views=ref["cr"]))):
        nrm, views = sub.get("nrm", E["n"]).float().contiguous(), sub.get("views", E["cr"]).float().contiguous()
        ft = torch.cat([torch.zeros(P, 1, device=cuda_dev), sub.get("feat", E["feat"]).float()], 1).contiguous()
        _, rgb_s = _render_tc(lib, N["rnet"], pts.contiguous(), nrm, views, ft)
        print("    with float64 %-14s shading max %.2e, %.2f %% above ELEM" % (
            name, float((rgb_s.double() - r64).abs()[keep].max()),
            100 * float(_elem_rows((rgb_s.double() - r64).abs(), r64)[keep].float().mean())))
    assert res["_rgb_elem"] <= 0.001
