"""The regulariser half of one optimisation step against a float64 twin that takes the engine's decisions
(train_step_twin.py): eikonal (grad_weight), offset and def_regu, one step per term with only that weight positive.
The surface-point terms (colour, weighted normal, the implicit term of propagateTmpPsGrad) and the template term are
not covered here.

Per term: the loss value (relative) and each parameter group's gradient as ||g - g64|| / ||g64|| (SDF, translator,
latent codes; the renderer, poses and translations get no gradient from these terms, on either side).  The engine's
figure is printed beside its bar and beside the figure of the same twin run in fp32.  Negative controls, each of which
must fail its bar: the twin without the ReLU replay, the def_regu GM scale c moved by 1 %, the translator's last
active positional-encoding band weight moved by 1e-3, and the SDF's softplus beta moved by 1 % (eikonal).  Two engine
runs of the same step are bit-identical."""
import pytest
import torch

import train_step_twin as TW

pytestmark = pytest.mark.gpu

_SCENE = {}


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
    return synth.Conf(base)


LOSS_KEY = {"eikonal": "grad_loss", "offset": "offset_loss", "def_regu": "def_loss"}
# bars: ~3x the first H100 measurement (DESIGN.md section 4, "training step vs float64")
# (def_regu: J = I + d offset / dp of a ReLU network is piecewise constant in the latent code, which gets no gradient)
BARS = {
    "eikonal": {"loss": 6e-6, "sdf": 1e-4},
    "offset": {"loss": 4e-7, "translator": 5e-6, "latent": 2e-5},
    "def_regu": {"loss": 3e-5, "translator": 4e-5},
}


def _engine(term, monkeypatch):
    net, data, rays, fids = scene()
    rec = TW.Record()
    with monkeypatch.context() as m:
        TW.record_engine(m, net, rec)
        out = TW.run_step(net, data, rays, fids, conf_for(term), torch.float32, True)
    return rec, out


def _twin(term, rec, dtype, monkeypatch, relu=True, c=0.5, pe_band_delta=0.0, sdf_beta=None):
    net, data = TW.make_twin(dtype)
    _, _, rays, fids = scene()
    with monkeypatch.context() as m:
        rr = TW.replay_twin(m, net, rec, dtype, relu=relu, pe_band_delta=pe_band_delta, sdf_beta=sdf_beta)
        out = TW.run_step(net, data, rays, fids, conf_for(term, c), dtype, False)
    return out, rr


def _figures(term, got, ref):
    """{"loss": rel err, group: ||g - g64|| / ||g64||} over the groups the term reaches."""
    (l, info, g), (l64, info64, g64) = got, ref
    k = LOSS_KEY[term]
    out = {"loss": abs(info[k] - info64[k]) / abs(info64[k])}
    for name, b in g64.items():
        nb = float(b.norm())
        if nb == 0.0:
            assert float(g[name].norm()) == 0.0, (term, name)
            continue
        out[name] = float((g[name] - b).norm()) / nb
    return out


@pytest.mark.parametrize("term", ["eikonal", "offset", "def_regu"])
def test_term_vs_float64_twin(term, monkeypatch):
    rec, eng = _engine(term, monkeypatch)
    ref, rr = _twin(term, rec, torch.float64, monkeypatch)
    f32, _ = _twin(term, rec, torch.float32, monkeypatch)
    e, t32 = _figures(term, eng, ref), _figures(term, f32, ref)
    print("\n[%s] samples replayed %d, translator ReLU decisions replayed %d, twin sign flips %d; repeated engine "
          "evaluations of the same points %d, ReLU decisions on which they disagree %d"
          % (term, len(rec.samples), rr.total, rr.flips, rec.relu_repeats, rec.relu_mismatch))
    assert rec.relu_mismatch == 0
    for k, v in e.items():
        print("[%s] %-10s engine %.2e  fp32 twin %.2e  bar %.0e" % (term, k, v, t32[k], BARS[term].get(k, 0)))
    assert set(e) == set(BARS[term]), (term, sorted(e))
    for k, v in e.items():
        assert v <= BARS[term][k], (term, k, v)
    # the engine run is deterministic
    _, eng2 = _engine(term, monkeypatch)
    assert eng2[0] == eng[0] and eng2[1][LOSS_KEY[term]] == eng[1][LOSS_KEY[term]]
    for name in eng[2]:
        assert torch.equal(eng[2][name], eng2[2][name]), (term, name)


@pytest.mark.parametrize("term,control", [("eikonal", "softplus beta +1%"),
                                          ("offset", "no ReLU replay"), ("def_regu", "no ReLU replay"),
                                          ("def_regu", "GM c +1%"), ("def_regu", "PE band weight +1e-3")])
def test_negative_controls_fail_their_bars(term, control, monkeypatch):
    rec, eng = _engine(term, monkeypatch)
    kw = {"no ReLU replay": dict(relu=False), "GM c +1%": dict(c=0.505),
          "PE band weight +1e-3": dict(pe_band_delta=1e-3), "softplus beta +1%": dict(sdf_beta=101.0)}[control]
    bad, _ = _twin(term, rec, torch.float64, monkeypatch, **kw)
    e = _figures(term, eng, bad)
    over = {k: v / BARS[term][k] for k, v in e.items()}
    print("\n[%s / %s] figure / bar: %s" % (term, control, ", ".join("%s %.1f" % kv for kv in over.items())))
    assert max(over.values()) > 1.0, (term, control, e)
