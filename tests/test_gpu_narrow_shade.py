"""The narrow (64-column) tile of the tensor-core layer kernel, and the reverse-mode SDF gradient of
ops.shade_and_render_tc (normals per component against the fp32 FFMA engine, colours as test_gpu_parity checks them,
and a negative control that drops the skip layer's part of the gradient).

Layers with N <= 64 -- the SDF's value-only output (N = 1), the translator's output (N = 3), the input gradient of a
reverse sweep (N = 39) -- are packed as [KC][planes][64 x 32] and run on n64 MMAs; N = 65 stays on the 256-column tile.
Every instantiation is checked against the float64 restatement of test_gpu_tc_contract at N = 8, 39, 64 and 65, with
M = 1, ragged row counts, skip columns and zero padding past the narrow tile, and (on the large geometry) m_dev below M
against sentinel-filled buffers, row independence and determinism."""
import pytest
import torch

from test_gpu_tc_contract import INSTANTIATIONS, INV_SQRT2, ACT, _Launch, _check_invariants, _check_layer, _inputs, _lib

NARROW_GEOMS = {
    # one point; skip columns appended right after the narrow tile's 8 columns, zeros up to K_next
    "M1_K64_N8_skip": dict(M=(1, 4), K=64, N=8, n=8, K_next=64, skip_n=20, scale=INV_SQRT2, out=(0, 8), rstash=False),
    # the reverse sweep's input gradient: next-layer chunks 2.. lie past the narrow tile (pack_skip_tail_kernel)
    "M333_K512_N39": dict(M=(333, 332), K=512, N=39, n=39, K_next=96, skip_n=0, scale=1.0, out=(0, 39), rstash=True),
    # the widest narrow layer, persistent over 394 row tiles; off-boundary output window
    "big_K256_N64_skip": dict(M=(50333, 50332), K=256, N=64, n=64, K_next=128, skip_n=39, scale=INV_SQRT2,
                              out=(5, 50), rstash=True),
    # one column past the narrow tile: the 256-column tile
    "M300_K96_N65": dict(M=(300, 300), K=96, N=65, n=65, K_next=128, skip_n=0, scale=1.0, out=(1, 64), rstash=True),
}
BIG = "big_K256_N64_skip"


def test_weight_pack_sizes_choose_the_tile():
    lib = _lib()
    kc_bytes = lambda bn: 2 * bn * 32 * 2          # noqa: E731  one k chunk of two bf16 planes
    for N in (1, 3, 39, 64):
        assert lib.sr_tc_weight_bytes(N, 512) == 16 * kc_bytes(64), N
    assert lib.sr_tc_weight_bytes(65, 512) == 16 * kc_bytes(256)
    assert lib.sr_tc_weight_bytes(257, 64) == 2 * 2 * kc_bytes(256)


@pytest.mark.gpu
@pytest.mark.parametrize("act,ch,mul", INSTANTIATIONS,
                         ids=["%s-%s-ch%d" % ("rev" if m else "fwd", ACT[a], c) for a, c, m in INSTANTIATIONS])
def test_narrow_tile_matches_fp64(cuda_dev, act, ch, mul):
    lib = _lib()
    for gi, (name, g) in enumerate(NARROW_GEOMS.items()):
        d = _inputs(cuda_dev, g, act, ch, mul, seed=1000 + 100 * gi + 10 * act + ch + (5 if mul else 0))
        L = _Launch(lib, cuda_dev, g, act, ch, mul, d)
        full = L.run()
        tag = "%s-%s-ch%d %s" % ("rev" if mul else "fwd", ACT[act], ch, name)
        _check_layer(lib, L, full, tag, controls=name == "M333_K512_N39")
        if name == BIG:
            _check_invariants(lib, L, full, tag)


# ---------------------------------------------------------------------------------------------------------------------
# shade_and_render_tc: grad f of the SDF in reverse mode
# ---------------------------------------------------------------------------------------------------------------------
# Normals, per component of the unit vector, against the fp32 FFMA engine (ops.shade_geometry).  Neither tensor-core
# path reaches 1e-5 on these inputs: the forward-tangent normals this change replaced measure 2.40e-5 and the
# reverse-mode ones 2.19e-5 (H100, DESIGN.md section 3.1b).  So the reverse-mode normals must be no worse than the
# forward tangents of the same engine, and within an absolute bar of twice that figure.
NORMAL_BAR = 5e-5


def _shade_inputs(dev):
    from helpers import RATIO, build_render, build_sdf_full, golden
    from test_gpu_parity import _deform_modules
    g, c, gs, gr = golden("deform.npz"), golden("cardinal.npz"), golden("sdf_full.npz"), golden("render.npz")
    comp, conds = _deform_modules(g, dev)
    sdf = build_sdf_full(gs).to(dev)
    rn = build_render(gr).to(dev)
    lbs = comp.defs[1].lbs_state()
    lbs.set_pose(conds[1][0], conds[1][1])
    return dict(full=sdf.fused(), dnet=comp.defs[0].fused(RATIO), rnet=rn.fused(RATIO), lbs=lbs, conds=conds,
                pts=torch.from_numpy(g["pts"]).to(dev), bi=torch.from_numpy(g["batch_inds"]).to(dev),
                rays=torch.from_numpy(c["rays"]).to(dev), golden=c)


@pytest.mark.gpu
def test_reverse_mode_normals_and_colours_match_ffma_engine(cuda_dev):
    import ctypes as C
    from helpers import rel_err
    from test_gpu_parity import FP_TOL
    from selfreconcode_b200 import ops
    s = _shade_inputs(cuda_dev)
    full, dnet, rnet, lbs, pts, bi, rays = (s[k] for k in ("full", "dnet", "rnet", "lbs", "pts", "bi", "rays"))
    n, cr, rgb, dp, ok = ops.shade_and_render_tc(full, dnet, lbs, rnet, pts, rays, bi, s["conds"][0])
    n2, cr2, ft, _, _ = ops.shade_geometry(full, dnet, lbs, pts, rays, bi, s["conds"][0], nfeat=256)
    rgb2 = ops.render_forward(rnet, pts, n2, cr2, ft)
    e_n = (n - n2).abs().max().item()
    e_rgb = rel_err(rgb.cpu().numpy(), rgb2.cpu().numpy())
    g4 = ops.tc_mlp_forward(full, pts, ch=4, n_out=1).view(-1, 4)[:, 1:]
    e_fwd = (torch.nn.functional.normalize(g4, dim=1) - n2).abs().max().item()
    print("reverse-mode normals: max |dn| %.2e (bar %.0e; forward tangents on the same engine %.2e) over %d points; "
          "rgb rel %.2e (bar %.0e)" % (e_n, NORMAL_BAR, e_fwd, pts.shape[0], e_rgb, 2 * FP_TOL))
    assert e_n <= e_fwd, "reverse mode less accurate than the forward tangents it replaced"
    assert e_n < NORMAL_BAR
    assert e_rgb < 2 * FP_TOL                                          # test_gpu_parity's colour check
    assert rel_err(cr.cpu().numpy(), s["golden"]["crays"]) < FP_TOL
    assert rel_err(dp.cpu().numpy(), s["golden"]["ds"]) < FP_TOL
    assert ok.all()
    # the cached work buffers: a smaller point count reuses them, a larger one than they hold grows them; every point's
    # result is its own
    c0 = s["conds"][0]
    for P2 in (100, 40 * pts.shape[0]):
        rep = (P2 + pts.shape[0] - 1) // pts.shape[0]
        p2, r2, b2 = (t.repeat(rep, *([1] * (t.dim() - 1)))[:P2] for t in (pts, rays, bi))
        n3, _, rgb3, _, _ = ops.shade_and_render_tc(full, dnet, lbs, rnet, p2, r2, b2, c0)
        m = min(P2, pts.shape[0])
        assert torch.equal(n3[:m], n[:m]) and torch.equal(rgb3[:m], rgb[:m]), P2
    # negative control: the same reverse sweep chained through the encoding without the skip layer's part
    lib = _lib()
    P = pts.shape[0]
    _, _, g_out = ops._sdf_grad_tc(lib, full, pts.contiguous(), P)
    d = full.desc
    pw = (C.c_float * 16)(*[d.pe_w[i] for i in range(16)])
    g_noskip = torch.empty(P, 3, device=cuda_dev)
    assert lib.sr_tc_embed_backward(ops._p(pts.contiguous()), P, d.multires, pw, 1, ops._p(g_out), g_out.shape[1], None, 0,
                                    ops._p(g_noskip), ops._stream()) == 0
    e_ctl = (torch.nn.functional.normalize(g_noskip, dim=1) - n2).abs().max().item()
    print("without the skip part: max |dn| %.2e (must exceed the bar)" % e_ctl)
    assert e_ctl > NORMAL_BAR and e_ctl > e_fwd
