"""CPU: pins the float64 restatement of the fp32 field engine (tests/ffma_ref.py) to the reference's golden vectors,
with the fixtures' own weights, and shows with negative controls that the same bars reject a restatement that drops
the skip connection's 1/sqrt(2), swaps sin and cos, ignores the band weights or stashes the skip input one layer late.

The bars are the GPU contract's (tests/test_gpu_ffma_contract.py): elem_err < 1e-4 on every output, norm_err < 1e-5
on values.  The goldens are fp32, so the measured errors here are the goldens' own rounding."""
import numpy as np
import torch

import ffma_ref as R
from helpers import (SMPL_PARENTS, build_render, build_sdf_full, build_sdf_small, build_translator, elem_err,
                     golden, norm_err, plain_params, sdf_params, wn_params)
from oracle import oracle as O

ELEM, NORM = 1e-4, 1e-5


def sdf_layers(params, skips):
    n = len(params)
    return [dict(v=v, g=g.view(-1), b=b, act=R.SP if l < n - 1 else R.NONE, skip=l in skips)
            for l, (v, g, b) in enumerate(params)]


def plain_layers(params, last_act, hidden_act=R.RELU):
    n = len(params)
    return [dict(v=w, g=None, b=b, act=hidden_act if l < n - 1 else last_act, skip=False)
            for l, (w, b) in enumerate(params)]


def wn_layers(params, last_act, hidden_act=R.RELU):
    n = len(params)
    return [dict(v=v, g=g.view(-1), b=b, act=hidden_act if l < n - 1 else last_act, skip=False)
            for l, (v, g, b) in enumerate(params)]


def _check(name, got, ref, value):
    e, n = elem_err(got, ref), norm_err(got, ref)
    print("%-22s elem %.2e  norm %.2e" % (name, e, n))
    assert e < ELEM, (name, e)
    if value:
        assert n < NORM, (name, n)
    return e


def test_sdf_small_value_grad_feature():
    g = golden("sdf_small.npz")
    layers = sdf_layers(sdf_params(build_sdf_small(g)), {2})
    pts = torch.from_numpy(g["pts"])
    for r in (1.0, 0.4):
        f, gr, out = R.sdf(layers, pts, 6, R.annealing_weights(6, r))
        _check("sdf_small f r%g" % r, f.numpy(), g["sdf_r%g" % r].reshape(-1), True)
        _check("sdf_small grad r%g" % r, gr.numpy(), g["grad_r%g" % r], False)
        _check("sdf_small feat r%g" % r, out[:, 1:].numpy(), g["feat_r%g" % r], True)


def test_sdf_full_value_grad_feature():
    g = golden("sdf_full.npz")
    layers = sdf_layers(sdf_params(build_sdf_full(g)), {4})
    f, gr, out = R.sdf(layers, torch.from_numpy(g["pts"]), 6, [1.0] * 6)
    _check("sdf_full f", f.numpy(), g["sdf"].reshape(-1), True)
    _check("sdf_full grad", gr.numpy(), g["grad"], False)
    _check("sdf_full feat", out[:, 1:].numpy(), g["feat"], True)


def deform_setup(g):
    """Translator layers, its PE band weights and the LBS inputs of deform.npz, all float64."""
    layers = plain_layers(plain_params(build_translator(g)), R.NONE)
    Js = torch.from_numpy(g["Js"]).double()
    ipi = O.init_pose_inverse(torch.from_numpy(g["apose"]).double(), Js, SMPL_PARENTS)
    A, posed = O.bone_transforms(torch.from_numpy(g["poses"]).double(), Js, SMPL_PARENTS, ipi)
    lbs = dict(ws=torch.from_numpy(g["ws"]).double(), bmin=torch.from_numpy(g["bmin"]).double(),
               bmax=torch.from_numpy(g["bmax"]).double(), A=A, trans=torch.from_numpy(g["trans"]).double())
    return layers, R.annealing_weights(6, float(g["def_ratio"])), lbs, posed


def deform_fn(layers, pe_w, lbs, conds, bi):
    def fn(x):
        p1 = x + R.translator_offset(layers, x, 6, pe_w, conds, bi)
        return O.lbs_forward(lbs["ws"], lbs["bmin"], lbs["bmax"], lbs["A"], lbs["trans"], p1, bi)
    return fn


def test_deformer_offset_and_jacobian():
    g = golden("deform.npz")
    layers, pe_w, lbs, posed = deform_setup(g)
    _check("bone posed joints", posed.numpy(), g["posed"], True)
    pts, bi = torch.from_numpy(g["pts"]), torch.from_numpy(g["batch_inds"])
    conds = torch.from_numpy(g["dcond"])
    off = R.translator_offset(layers, pts.double(), 6, pe_w, conds, bi)
    _check("translator offset", off.numpy(), g["offset"], True)
    d, J = R.jacobian(deform_fn(layers, pe_w, lbs, conds, bi), pts)
    _check("deformed point", d.numpy(), g["d"], True)
    _check("deformer jacobian", J.numpy(), g["jac"], False)


def test_cardinal_rays():
    g, c = golden("deform.npz"), golden("cardinal.npz")
    layers, pe_w, lbs, _ = deform_setup(g)
    pts, bi = torch.from_numpy(g["pts"]).double(), torch.from_numpy(g["batch_inds"])
    fn = deform_fn(layers, pe_w, lbs, torch.from_numpy(g["dcond"]), bi)
    cr, ds, _, ok = O.cardinal_rays(fn, pts, torch.from_numpy(c["rays"]).double())
    assert bool(ok.all())
    _check("cardinal rays", cr.numpy(), c["crays"], True)
    _check("cardinal D(p)", ds.numpy(), c["ds"], True)


def test_render_net():
    g = golden("render.npz")
    layers = wn_layers(wn_params(build_render(g)), R.TANH)
    rgb, margin = R.render(layers, torch.from_numpy(g["pts"]), torch.from_numpy(g["normals"]),
                           torch.from_numpy(g["views"]), torch.from_numpy(g["feat"]), 4, [1.0] * 4)
    _check("render rgb", rgb.numpy(), g["rgb"], True)
    assert float(margin.min()) > 0.0


def test_negative_controls_fail_the_bars():
    """Each variant differs from the engine's arithmetic by one term; its error must exceed the elementwise bar."""
    gs, gf = golden("sdf_small.npz"), golden("sdf_full.npz")
    small = sdf_layers(sdf_params(build_sdf_small(gs)), {2})
    full = sdf_layers(sdf_params(build_sdf_full(gf)), {4})
    ps, pf = torch.from_numpy(gs["pts"]), torch.from_numpy(gf["pts"])
    cases = {
        "skip without 1/sqrt(2)": (R.sdf(full, pf, 6, [1.0] * 6, skip_scale=1.0), gf["sdf"], gf["grad"]),
        "sin and cos swapped": (R.sdf(small, ps, 6, [1.0] * 6, swap_sincos=True), gs["sdf_r1"], gs["grad_r1"]),
        "band weights ignored": (R.sdf(small, ps, 6, [1.0] * 6), gs["sdf_r0.4"], gs["grad_r0.4"]),
        "skip stash one layer late": (R.sdf(full, pf, 6, [1.0] * 6, late_stash=True), gf["sdf"], gf["grad"]),
    }
    for name, ((f, gr, _), f_ref, g_ref) in cases.items():
        ef, eg = elem_err(f.numpy(), f_ref.reshape(-1)), elem_err(gr.numpy(), g_ref)
        print("negative control %-26s elem f %.2e  grad %.2e" % (name, ef, eg))
        assert ef > 10 * ELEM and eg > 10 * ELEM, name
