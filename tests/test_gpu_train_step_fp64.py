"""Each loss term of one optimisation step against a float64 twin that takes the engine's decisions
(train_step_twin.py), one step per term with only that weight positive: eikonal (grad_weight), offset, def_regu,
colour, weighted normal, and the mix of the shipped coarse level's ray weights.  The colour and normal terms run the
surface-point branch and with it the implicit term of propagateTmpPsGrad.  The template (point-cloud silhouette and
mesh) term is not covered here.

Per term: the loss value (relative), dL/dTmpPs, and each parameter group's gradient as ||g - g64|| / ||g64|| (SDF,
translator, renderer, poses, translations, latent codes), once for the gradient of loss.backward() (the direct part)
and once for that of propagateTmpPsGrad alone (the implicit part, "implicit <group>").  A group the term does not reach
in float64 must get exactly zero on the engine.  The engine's figure is printed beside its bar and beside the figure
of the same twin run in fp32.  Rays whose step takes a decision the twin cannot replay (train_step_twin.keep_mask) are
removed from both runs; at most 1 % of the converged rays.  Negative controls, each of which must fail its bar: the
twin without the ReLU replay (translator; renderer, when the replay flipped a decision), the def_regu GM scale c moved
by 1 %, the translator's or the renderer's last active positional-encoding band weight moved by 1e-3, the SDF's
softplus beta moved by 1 % (eikonal, mix), the root joint's pose moved by 1e-4 rad, one entry of the deformer Jacobian
scaled by 1 + 1e-3, and the colour and normal losses taken as one mean over all rays instead of the mean of per-frame
means; FAILS names the bars each must fail, and together they cover every bar of the surface terms.  Two engine runs of
the same step are bit-identical."""
import pytest
import torch

import train_step_twin as TW

pytestmark = pytest.mark.gpu

_SCENE = {}
_SURFACE = {}

SURFACE_TERMS = ("colour", "normal", "mix")


def scene():
    if not _SCENE:
        import test_optim_step_gpu as S
        net, data, rays, fids = S.build()
        _SCENE.update(net=net, data=data, rays=rays, fids=fids)
    return _SCENE["net"], _SCENE["data"], _SCENE["rays"], _SCENE["fids"]


def conf_for(term, c=0.5):
    from selfreconcode_b200 import synth
    base = dict(grad_weight=0.0, color_weight=0.0, normal_weight=0.0)
    if term == "eikonal":
        base["grad_weight"] = 0.1
    elif term == "offset":
        base["offset_weight"] = 0.05
    elif term == "def_regu":
        base["def_regu"] = dict(weight=2.0, c=c)
    elif term == "colour":
        base["color_weight"] = 0.5
    elif term == "normal":
        base.update(normal_weight=0.1, weighted_normal=True)
    elif term == "mix":
        # the shipped coarse level's ray weights; its offset_weight 0 only logs the offset term, so it is left out
        base.update(grad_weight=1.0, color_weight=0.5, normal_weight=0.1, weighted_normal=True,
                    def_regu=dict(weight=0.1, c=c))
    return synth.Conf(base)


LOSS_KEY = {"eikonal": "grad_loss", "offset": "offset_loss", "def_regu": "def_loss", "colour": "color_loss",
            "normal": "normal_loss", "mix": None}      # None: the step's total loss
# bars: ~3x the first H100 measurement (DESIGN.md section 4, "training step vs float64")
# (def_regu: J = I + d offset / dp of a ReLU network is piecewise constant in the latent code, which gets no gradient)
BARS = {
    "eikonal": {"loss": 6e-6, "sdf": 1e-4},
    "offset": {"loss": 4e-7, "translator": 5e-6, "latent": 2e-5},
    "def_regu": {"loss": 3e-5, "translator": 4e-5},
    "colour": {"loss": 5e-7, "TmpPs": 6e-5, "sdf": 6e-5, "translator": 5e-5, "renderer": 2e-5, "poses": 6e-5,
               "latent": 5e-5, "implicit sdf": 1e-4, "implicit translator": 8e-5, "implicit poses": 7e-5,
               "implicit trans": 1e-4, "implicit latent": 1e-4},
    "normal": {"loss": 4e-6, "TmpPs": 6e-5, "sdf": 8e-5, "translator": 9e-6, "poses": 5e-6, "latent": 3e-5,
               "implicit sdf": 5e-5, "implicit translator": 4e-5, "implicit poses": 4e-5, "implicit trans": 4e-5,
               "implicit latent": 6e-5},
    # (mix sdf: the eikonal term at grad_weight 1 dominates it, with the second-order softplus(100) error of the eikonal
    # row above)
    "mix": {"loss": 6e-7, "TmpPs": 6e-5, "sdf": 2e-4, "translator": 1e-5, "renderer": 2e-5, "poses": 5e-6,
            "latent": 3e-5, "implicit sdf": 5e-5, "implicit translator": 4e-5, "implicit poses": 4e-5,
            "implicit trans": 5e-5, "implicit latent": 4e-5},
}


def _engine(term, monkeypatch, keep=None):
    net, data, rays, fids = scene()
    rec = TW.Record()
    with monkeypatch.context() as m:
        TW.record_engine(m, net, rec, surface=term in SURFACE_TERMS, keep=keep)
        out = TW.run_step(net, data, rays, fids, conf_for(term), torch.float32, True)
    return rec, out


def _gt_colours():
    net, data, rays, fids = scene()
    img, _ = TW.images(fids.numel(), data.H, data.W, torch.float64)
    return img[rays["batch_inds"].cuda(), rays["rows"].cuda(), rays["cols"].cuda()]


def _surface_engine(term, monkeypatch):
    """A first engine run finds the rays whose decisions the twin cannot replay; a second one runs without them.
    -> (record, Step, {reason: rays excluded}, converged rays of the first run), kept per term."""
    if term not in _SURFACE:
        rec1, _ = _engine(term, monkeypatch)
        keep, counts, n_conv = TW.keep_mask(rec1, _gt_colours())
        rec, out = _engine(term, monkeypatch, keep=keep)
        assert torch.equal(rec.trace[0][0], rec1.trace[0][0])            # the second run traces the same points
        assert torch.equal(rec.trace[0][1], rec1.trace[0][1] & keep)
        _SURFACE[term] = (rec, out, counts, n_conv)
    return _SURFACE[term]


def _twin(term, rec, dtype, monkeypatch, c=0.5, **kw):
    net, data = TW.make_twin(dtype)
    _, _, rays, fids = scene()
    with monkeypatch.context() as m:
        rr = TW.replay_twin(m, net, rec, dtype, **kw)
        out = TW.run_step(net, data, rays, fids, conf_for(term, c), dtype, False)
    return out, rr


def _rel(a, b):
    return float((a - b).norm()) / float(b.norm())


def _figures(term, got, ref):
    """{"loss": rel err, "TmpPs": dL/dTmpPs, group / "implicit " group: ||g - g64|| / ||g64||} over what the term
    reaches in float64."""
    k = LOSS_KEY[term]
    l, l64 = (got.loss, ref.loss) if k is None else (got.info[k], ref.info[k])
    out = {"loss": abs(l - l64) / abs(l64)}
    if ref.dtmp is not None:
        out["TmpPs"] = _rel(got.dtmp, ref.dtmp)
    for prefix, g, g64 in (("", got.direct, ref.direct), ("implicit ", got.implicit, ref.implicit)):
        for name, b in g64.items():
            if float(b.norm()) == 0.0:
                assert float(g[name].norm()) == 0.0, (term, prefix + name)
                continue
            out[prefix + name] = _rel(g[name], b)
    return out


def _bar_ratios(term, e):
    return {k: v / BARS[term][k] if k in BARS[term] else float("inf") for k, v in e.items()}


@pytest.mark.parametrize("term", ["eikonal", "offset", "def_regu"] + list(SURFACE_TERMS))
def test_term_vs_float64_twin(term, monkeypatch):
    surface = term in SURFACE_TERMS
    if surface:
        rec, eng, counts, n_conv = _surface_engine(term, monkeypatch)
    else:
        rec, eng = _engine(term, monkeypatch)
    ref, rr = _twin(term, rec, torch.float64, monkeypatch)
    f32, _ = _twin(term, rec, torch.float32, monkeypatch)
    e, t32 = _figures(term, eng, ref), _figures(term, f32, ref)
    print("\n[%s] samples replayed %d, translator ReLU decisions replayed %d, twin sign flips %d; repeated engine "
          "evaluations of the same points %d, ReLU decisions on which they disagree %d"
          % (term, len(rec.samples), rr.tr.total, rr.tr.flips, rec.relu_repeats, rec.relu_mismatch))
    if surface:
        print("[%s] renderer ReLU decisions replayed %d, twin sign flips %d; converged rays %d, excluded %s; invInfo "
              "engine %s twin %s" % (term, rr.rn.total if rr.rn else 0, rr.rn.flips if rr.rn else 0, n_conv, counts,
                                     eng.info["invInfo"], ref.info["invInfo"]))
    for k, v in e.items():
        print("[%s] %-20s engine %.2e  fp32 twin %.2e  bar %.0e" % (term, k, v, t32[k], BARS[term].get(k, 0)))
    assert rec.relu_mismatch == 0
    if surface:
        assert counts["any"] <= 0.01 * n_conv, counts
        conv = eng.info["rayInfo"][1]
        assert conv == n_conv - counts["any"] and ref.info["rayInfo"] == eng.info["rayInfo"]
        assert eng.info["invInfo"] == ref.info["invInfo"] and eng.info["invInfo"][0] == conv, (eng.info, ref.info)
        if rec.colors:
            # no colour component of a kept ray sits within the kink margin on one side and across it on the other
            assert len(rec.colors) == 1 and len(rr.colors) == 1
            dc = float((rec.colors[0].double() - rr.colors[0].double()).abs().max())
            print("[%s] max |c_engine - c_twin| %.2e (kink margin %.0e)" % (term, dc, TW.KINK_MARGIN))
            assert dc < TW.KINK_MARGIN
    # the engine run is deterministic
    _, eng2 = _engine(term, monkeypatch, keep=rec.trace[0][1] if surface else None)
    assert eng2.loss == eng.loss and eng2.info == eng.info
    for part in ("direct", "implicit"):
        for name in getattr(eng, part):
            assert torch.equal(getattr(eng, part)[name], getattr(eng2, part)[name]), (term, part, name)
    assert (eng.dtmp is None) == (eng2.dtmp is None) and (eng.dtmp is None or torch.equal(eng.dtmp, eng2.dtmp))
    assert set(e) == set(BARS[term]), (term, sorted(e))
    for k, v in e.items():
        assert v <= BARS[term][k], (term, k, v)


CONTROLS = {"no ReLU replay": dict(relu=False), "GM c +1%": dict(c=0.505),
            "PE band weight +1e-3": dict(pe_band_delta=1e-3), "softplus beta +1%": dict(sdf_beta=101.0),
            "renderer PE band weight +1e-3": dict(render_pe_delta=1e-3), "root pose +1e-4 rad": dict(pose_delta=1e-4),
            "Jacobian entry x(1+1e-3)": dict(jac_scale=1.0 + 1e-3), "no renderer ReLU replay": dict(render_relu=False),
            "one mean over all rays": dict(pooled_mean=True)}
_IMPLICIT = tuple("implicit " + g for g in ("sdf", "translator", "poses", "trans", "latent"))
# the bars each control must fail, beyond failing one: together they cover every bar of the surface terms
FAILS = {("colour", "one mean over all rays"): ("loss", "sdf"),
         ("colour", "renderer PE band weight +1e-3"): ("TmpPs", "translator", "renderer", "poses", "latent"),
         ("colour", "Jacobian entry x(1+1e-3)"): _IMPLICIT,
         ("normal", "Jacobian entry x(1+1e-3)"): tuple(BARS["normal"]),
         ("mix", "softplus beta +1%"): ("sdf",),
         ("mix", "renderer PE band weight +1e-3"): ("renderer",),
         ("mix", "Jacobian entry x(1+1e-3)"): ("loss", "TmpPs", "translator", "poses", "latent") + _IMPLICIT}


@pytest.mark.parametrize("term,control", [("eikonal", "softplus beta +1%"),
                                          ("offset", "no ReLU replay"), ("def_regu", "no ReLU replay"),
                                          ("def_regu", "GM c +1%"), ("def_regu", "PE band weight +1e-3")]
                         + [(t, c) for t in ("colour", "mix") for c in ("renderer PE band weight +1e-3",
                                                                       "no renderer ReLU replay")]
                         + [(t, c) for t in SURFACE_TERMS for c in ("root pose +1e-4 rad", "Jacobian entry x(1+1e-3)")]
                         + [("colour", "one mean over all rays"), ("mix", "softplus beta +1%")])
def test_negative_controls_fail_their_bars(term, control, monkeypatch):
    if term in SURFACE_TERMS:
        rec, eng = _surface_engine(term, monkeypatch)[:2]
    else:
        rec, eng = _engine(term, monkeypatch)
    bad, rr = _twin(term, rec, torch.float64, monkeypatch, **CONTROLS[control])
    e = _figures(term, eng, bad)
    over = _bar_ratios(term, e)
    print("\n[%s / %s] figure (figure / bar): %s" % (term, control, ", ".join("%s %.2e (%.1f)" % (k, e[k], over[k])
                                                                             for k in e)))
    if control == "no renderer ReLU replay" and rr.rn.flips == 0:
        print("[%s / %s] the replay flipped no renderer decision: nothing to control" % (term, control))
        return
    assert max(over.values()) > 1.0, (term, control, e)
    for k in FAILS.get((term, control), ()):
        assert over[k] > 1.0, (term, control, k, e[k])


def test_every_surface_bar_has_a_failing_control():
    for term in SURFACE_TERMS:
        covered = set(k for (t, _), keys in FAILS.items() if t == term for k in keys)
        assert covered == set(BARS[term]), (term, sorted(set(BARS[term]) - covered))


@pytest.mark.parametrize("term", ["colour", "normal"])
def test_twin_refuses_fp32_entry_points(term, monkeypatch):
    """With the twin's deformer reporting itself fusable, propagateTmpPsGrad (colour) and compute_deformed_normals
    (weighted normal) take their no-graph fp32 branches; the twin refuses them instead of promoting their results."""
    rec = _surface_engine(term, monkeypatch)[0]
    net, data = TW.make_twin(torch.float64)
    _, _, rays, fids = scene()
    with monkeypatch.context() as m:
        TW.replay_twin(m, net, rec, torch.float64)
        m.setattr(net.deformer, "_fusable", lambda: True)
        with pytest.raises(RuntimeError, match="fp32 field-engine entry point"):
            TW.run_step(net, data, rays, fids, conf_for(term), torch.float64, False)
