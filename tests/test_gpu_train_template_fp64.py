"""The template term of one optimisation step (OptimNetwork.forward -> computeTmpPcLoss: the soft point silhouette's
IoU against the dilated gt mask, the mesh regularisers, the def_consistent GM term, the inner backward and SGD step on
TmpVs, and the |f| tie of the SDF to the moved template) against the float64 twin of train_step_twin.py, end to end:
forward() -> loss.backward() -> propagateTmpPsGrad, with the level set by utils.set_hierarchical_config.  One step per
case, each with one pc_weight block; every ray weight 0 and no surface rays except in step:

  mask      mask_weight 1                                  mask_loss, displacement, translator / poses / trans / latent
  mesh      laplacian / edge / normal weights > 0          the three values, displacement; every group exactly 0
  defconst  def_consistent 0.6 / c 0.01 (config.conf)      defconst_loss, displacement, translator / poses / latent
  sdf       weight 60 (the template does not move)         pc_loss_sdf, SDF
  shipped   config.conf's coarse block                     all of the above
  step      shipped + the shipped coarse ray mix, surface  all of the above, and what test_gpu_train_step_fp64's mix
            rays on                                        reports: ray losses, dL/dTmpPs, renderer, implicit part

Per case: every value the step reports (relative), the step's loss (relative, where it is not 0), the inner SGD step's
displacement -lr dL/dTmpVs as ||d - d64|| / ||d64||, each parameter group's gradient as ||g - g64|| / ||g64|| (after
backward, and of propagateTmpPsGrad alone: "implicit <group>") and dL/dTmpPs; a group (or displacement) that is 0 in
float64 must be exactly 0 on the engine.  Under defconst the translation gradient cancels analytically: dv and the
rigid LBS add the translation by the same broadcast op, so its two paths cancel exactly on both sides and the group is
held to that exact-zero rule.  The engine's figure is printed beside the fp32 twin's and the bar.  Point radius
0.04 at 96x96 (mask, mesh: the gt mask dilated by 2 pixels) and 0.01 (the others: no dilation).  forward()'s glue (the
gt-mask selection of the seed pixels, the sample_pix subsampling, the extra template points) is restated and checked
on both runs (train_step_twin.forward_glue); in step those pixels are the rays the surface terms train on.  The
engine's sign of the |f| tie is replayed, and must be the twin's own wherever |f64| >= SIGN_BOUND.

Template vertices whose term takes a decision the twin cannot replay (train_step_twin.template_borderline) are moved
by a fixed step in a second engine run, which finds none left (further runs would move the new ones, at most
MOVE_ROUNDS); the twin replays that template.  In step a further run then drops the rays keep_mask finds.  Negative
controls (CONTROLS; FAILS names the bars each must fail, together every bar; MAY_PASS those that cannot change this
scene, and why): the silhouette radius +1 %, the dilation one pixel wider, mesh_reg_ref's own switches and the normal
term without the minus sign of -n_j, def_consistent c +1 %, SGD lr +1 %, the inner backward's deformer gradients
dropped (the reference keeps them for the outer optimiser), the twin's own |f| instead of the engine's sign (skipped
when the replay flips no sign), the root pose +1e-4 rad, the translator's last active PE band +1e-3, the SDF's softplus
beta +1 %, and in step the surface terms' controls of test_gpu_train_step_fp64.py.  The kernel's K truncation is not
checked here: the mask case has up to 276 points on a pixel against K = 50, but the 50 nearest already drive
1 - prod(1 - w) to 1 there, so no figure changes without the truncation; test_gpu_points_silhouette.py pins it.  Two
engine runs of the same step are bit-identical."""
import copy

import numpy as np
import pytest
import torch

import helpers as H
import points_silhouette_ref as PS
import train_step_twin as TW

pytestmark = pytest.mark.gpu

_SCENE = {}
_ENGINE = {}

CASES = ("mask", "mesh", "defconst", "sdf", "shipped", "step")
RADIUS = {"mask": 0.04, "mesh": 0.04, "defconst": 0.01, "sdf": 0.01, "shipped": 0.01, "step": 0.01}
K = 50                  # update_hierarchical_config's points_per_pixel
MOVE_ROUNDS = 4         # engine runs that may find borderline vertices
SAMPLE_PIX = 200        # per frame: below the seed's pixel count, so forward() subsamples it
_OFF = dict(laplacian_weight=-10., edge_weight=-10., norm_weight=-0.001)     # config.conf's coarse mesh weights
PC = {"mask": dict(weight=0., mask_weight=1., **_OFF),
      "mesh": dict(weight=0., mask_weight=0., laplacian_weight=0.1, edge_weight=1.0, norm_weight=0.01),
      "defconst": dict(weight=0., mask_weight=0., def_consistent=dict(weight=0.6, c=0.01)),
      "sdf": dict(weight=60., mask_weight=0.),
      "shipped": dict(weight=60., mask_weight=1., def_consistent=dict(weight=0.6, c=0.01), **_OFF)}
PC["step"] = PC["shipped"]
# the shipped coarse level's ray weights (test_gpu_train_step_fp64's mix), with surface rays, in the step case
RAY_MIX = dict(grad_weight=1.0, color_weight=0.5, normal_weight=0.1, weighted_normal=True, def_regu=dict(weight=0.1,
                                                                                                         c=0.5))
VALUES = ("mask_loss", "lap_loss", "edge_loss", "norm_loss", "defconst_loss")
RAY_VALUES = ("grad_loss", "def_loss", "color_loss", "normal_loss")
# |f64| at every vertex where the twin's own sign differs from the engine's: ~3x the measured 8.7e-7, below the
# tensor-core engine's own error on these vertices (up to 1.2e-5), so a sign taken on the tensor-core value instead of
# the refine band's fp32 re-evaluation fails it
SIGN_BOUND = 3e-6

# bars: ~3x the first H100 measurement (DESIGN.md section 4, "template term vs float64")
# (pc_loss_sdf, and the loss of sdf and shipped it makes: a mean of sign(f) f over vertices on the zero set, ~3e-4, so
# its relative figure is the engine's absolute value error over that mean; the tensor-core and the fp32 values carry
# the same, see DESIGN.md.  shipped poses / trans: the plain fp32 twin measures the same 1.1e-4 / 1.0e-4)
BARS = {
    "mask": {"mask_loss": 3e-7, "pc_loss_sdf": 7e-3, "displacement": 1e-4, "translator": 1.1e-4, "poses": 7e-5,
             "trans": 1.2e-4, "latent": 1.1e-4},
    "mesh": {"mask_loss": 3e-7, "lap_loss": 1e-7, "edge_loss": 7e-8, "norm_loss": 2e-8, "pc_loss_sdf": 8e-3,
             "displacement": 1e-7},
    "defconst": {"mask_loss": 6e-7, "defconst_loss": 4e-7, "pc_loss_sdf": 7e-3, "displacement": 2e-5,
                 "translator": 6e-6, "poses": 2e-5, "latent": 3e-5},
    "sdf": {"loss": 8e-3, "mask_loss": 5e-7, "pc_loss_sdf": 8e-3, "sdf": 4e-5},
    # (step: the template figures as shipped's, plus test_gpu_train_step_fp64's mix figures on forward()'s pixel set)
    "step": {"loss": 1.3e-4, "mask_loss": 6e-7, "defconst_loss": 4e-7, "grad_loss": 1e-5, "def_loss": 3.3e-5,
             "color_loss": 1.5e-7, "normal_loss": 1.4e-6, "TmpPs": 5e-5, "pc_loss_sdf": 6e-3, "displacement": 1.2e-4,
             "sdf": 5e-5, "translator": 2e-4, "renderer": 2.4e-5, "poses": 4e-4, "trans": 4e-4, "latent": 2e-4,
             "implicit sdf": 7.5e-5, "implicit translator": 5e-5, "implicit poses": 7e-5, "implicit trans": 7e-5,
             "implicit latent": 5.5e-5},
    "shipped": {"loss": 6e-3, "mask_loss": 6e-7, "defconst_loss": 4e-7, "pc_loss_sdf": 6e-3, "displacement": 1.2e-4,
                "sdf": 4e-5, "translator": 2e-4, "poses": 4e-4, "trans": 4e-4, "latent": 2e-4},
}


def gt_mask(N, Hh, Ww):
    """A seeded gt mask: an ellipse off the body's centre with 2 % of its pixels flipped."""
    g = torch.Generator().manual_seed(13)
    yy, xx = torch.meshgrid(torch.arange(Hh).double(), torch.arange(Ww).double(), indexing="ij")
    m = (((yy - 0.55 * Hh) / (0.3 * Hh)) ** 2 + ((xx - 0.45 * Ww) / (0.2 * Ww)) ** 2 < 1).double()
    m = m.expand(N, Hh, Ww).clone()
    flip = torch.rand(N, Hh, Ww, generator=g) < 0.02
    m[flip] = 1.0 - m[flip]
    return m


def scene():
    """test_optim_step_gpu.build()'s net with the built-in mesh rasteriser as maskRender (so that the level installs
    the built-in point renderer), and the step's images."""
    if not _SCENE:
        import test_optim_step_gpu as S
        H.dropin()
        from model.raster import MeshRasterizer, RasterSettings, SilhouetteRenderer
        net, data, _, fids = S.build()
        net.maskRender = SilhouetteRenderer(MeshRasterizer(net.maskRender.rasterizer.cameras,
                                                           RasterSettings((data.H, data.W))))
        img, nrm = TW.images(fids.numel(), data.H, data.W, torch.float64)
        datas = {"img": img, "normal": nrm, "mask": gt_mask(fids.numel(), data.H, data.W).to(TW.DEV)}
        _SCENE.update(net=net, data=data, fids=fids, datas=datas)
    return _SCENE["net"], _SCENE["data"], _SCENE["fids"], _SCENE["datas"]


def conf_for(case, c=None):
    from selfreconcode_b200 import synth
    pc = copy.deepcopy(PC[case])
    if c is not None:
        pc["def_consistent"]["c"] = c
    loss = dict(grad_weight=0., color_weight=0., normal_weight=0., sample_pix_num=SAMPLE_PIX, pc_weight=pc)
    if case == "step":
        loss.update(copy.deepcopy(RAY_MIX))
    return synth.Conf(train=dict(coarse=dict(point_render=dict(radius=RADIUS[case], remesh_intersect=30,
                                                                batch_size=2))),
                      loss_coarse=loss)


def _engine(case, monkeypatch, move=None, keep=None):
    net, data, fids, datas = scene()
    rec = TW.Record()
    with monkeypatch.context() as m:
        TW.record_engine(m, net, rec, surface=case == "step", keep=keep)
        hold = TW.record_template(m, net, rec, move)
        TW.forward_glue(m, net, rec)
        out = TW.run_forward(net, data, datas, fids, conf_for(case), torch.float32, True, hold)
    return rec, out


def _engine_case(case, monkeypatch):
    """A first engine run finds the template vertices whose decisions the twin cannot replay; the next one runs with
    them moved, and so on (a moved point can become the K-th of a crowded pixel) until a run finds none, at most
    MOVE_ROUNDS.  With surface rays (step) a further run then drops the rays whose step takes a decision the twin
    cannot replay (train_step_twin.keep_mask over forward()'s pixel set).  -> (record, TStep, [{reason: vertices} per
    run], move, (keep, {reason: rays}, converged rays) or None), kept per case."""
    if case not in _ENGINE:
        rec, out = _engine(case, monkeypatch)
        tmp0 = rec.tmp
        steps = None
        counts = []
        for _ in range(MOVE_ROUNDS):
            found, c = TW.template_borderline(rec)
            counts.append(c)
            if c["any"] == 0:
                break
            steps = found.int() if steps is None else steps + found.int()
            rec, out = _engine(case, monkeypatch, move=steps)
            assert torch.equal(rec.tmp[1], tmp0[1])
        rays = None
        if case == "step":
            _, _, _, datas = scene()
            bi, ri, ci = rec.pixels
            keep, kc, n_conv = TW.keep_mask(rec, datas["img"][bi, ri, ci])
            rec1 = rec
            rec, out = _engine(case, monkeypatch, move=steps, keep=keep)
            assert all(torch.equal(a, b) for a, b in zip(rec.pixels, rec1.pixels))
            assert torch.equal(rec.trace[0][0], rec1.trace[0][0])       # the kept rays trace the same points
            assert torch.equal(rec.trace[0][1], rec1.trace[0][1] & keep)
            assert TW.template_borderline(rec)[1]["any"] == 0
            rays = (keep, kc, n_conv)
        _ENGINE[case] = (rec, out, counts, steps, rays)
    return _ENGINE[case]


_TWIN_KW = ("relu", "pe_band_delta", "pose_delta", "sdf_beta", "render_relu", "render_pe_delta", "jac_scale",
            "pooled_mean")


def _twin(case, rec, dtype, monkeypatch, c=None, **kw):
    net, data = TW.make_twin(dtype, mesh_raster=True)
    _, _, fids, datas = scene()
    twin_kw = {k: kw.pop(k) for k in _TWIN_KW if k in kw}
    with monkeypatch.context() as m:
        rr = TW.replay_twin(m, net, rec, dtype, **twin_kw)
        hold = TW.replay_template(m, net, rec, dtype, **kw)
        hold.glue = TW.forward_glue(m, net, rec, replay_extra=True)
        hold.rr = rr
        out = TW.run_forward(net, data, datas, fids, conf_for(case, c), dtype, False, hold)
    return out, hold


def _rel(a, b):
    return float((a - b).norm()) / float(b.norm())


def _figures(case, got, ref):
    """{value / "loss" / "displacement" / group: relative error} over what the case reaches in float64."""
    out = {}
    if ref.loss != 0.0:
        out["loss"] = abs(got.loss - ref.loss) / abs(ref.loss)
    else:
        assert got.loss == 0.0, (case, got.loss)
    for k in VALUES:
        if k in ref.info["pc_loss"]:
            out[k] = abs(got.info["pc_loss"][k] - ref.info["pc_loss"][k]) / abs(ref.info["pc_loss"][k])
    if case == "step":
        for k in RAY_VALUES:
            out[k] = abs(got.info[k] - ref.info[k]) / abs(ref.info[k])
    if ref.dtmp is not None:
        out["TmpPs"] = _rel(got.dtmp, ref.dtmp)
    out["pc_loss_sdf"] = abs(got.info["pc_loss_sdf"] - ref.info["pc_loss_sdf"]) / abs(ref.info["pc_loss_sdf"])
    if float(ref.disp.norm()) == 0.0:
        assert float(got.disp.norm()) == 0.0, (case, "displacement")
    else:
        out["displacement"] = _rel(got.disp, ref.disp)
    for prefix, gs, gs64 in (("", got.direct, ref.direct), ("implicit ", got.implicit, ref.implicit)):
        for name, b in gs64.items():
            g = gs[name]
            if float(b.norm()) == 0.0:
                if float(g.norm()) != 0.0:
                    out[prefix + name] = float("inf")    # a group the term does not reach must get exactly zero
                continue
            out[prefix + name] = _rel(g, b)
    return out


def _bar_ratios(case, e):
    return {k: v / BARS[case][k] if k in BARS[case] else float("inf") for k, v in e.items()}


def _silhouette_stats(rec, datas):
    """(max covering points on a pixel, pixels the silhouette covers inside the gt mask, outside it) of the engine's
    own screen points."""
    pts, Hh, Ww, r, K_ = rec.sil[0]
    ndc = PS.screen_to_ndc(pts.double().cpu().numpy(), Hh, Ww)
    R = PS.rasterize(ndc, Hh, Ww, r, None)
    m = PS.silhouette(ndc, Hh, Ww, r, K_) > 0.5
    gt = datas["mask"].cpu().numpy() > 0.5
    return int(R["n_cover"].max()), int((m & gt).sum()), int((m & ~gt).sum())


@pytest.mark.parametrize("case", CASES)
def test_template_term_vs_float64_twin(case, monkeypatch):
    rec, eng, counts, move, rays = _engine_case(case, monkeypatch)
    ref, h64 = _twin(case, rec, torch.float64, monkeypatch)
    f32, h32 = _twin(case, rec, torch.float32, monkeypatch)
    e, t32 = _figures(case, eng, ref), _figures(case, f32, ref)
    _, _, fids, datas = scene()
    ncov, inside, outside = _silhouette_stats(rec, datas)
    Hh, Ww = datas["mask"].shape[1:]
    dil = int(np.round(RADIUS[case] / 2. * float(min(Hh, Ww)) / 1.2))
    print("\n[%s] template %d vertices, %d faces; radius %g (gt dilation %d px); max points on a pixel %d (K %d); "
          "silhouette pixels inside / outside the gt mask %d / %d; seed pixels %d"
          % (case, rec.tmp[0].shape[0], rec.tmp[1].shape[0], RADIUS[case], dil, ncov, K, inside, outside,
             rec.seed[0].numel()))
    N, V = fids.numel(), rec.tmp[0].shape[0]
    tkey = ("translator", TW.points_key(rec.tmp[0][None].expand(N, V, 3)))
    flip_max = float(h64.flip_f64.max()) if h64.sign_flips else 0.0
    print("[%s] borderline vertices per engine run %s, vertices moved %d; translator ReLU decisions on the template "
          "recorded %d (all evaluations: %d repeats, %d mismatches); |f| tie sign flips %s of %d, max |f64| there %.2e"
          % (case, counts, rec.moved, sum(int(x.numel()) for x in rec.relu[tkey]), rec.relu_repeats,
             rec.relu_mismatch, h64.sign_flips, h64.sign_total, flip_max))
    if rays is not None:
        print("[%s] rays of forward()'s pixel set %d, converged %d, excluded %s; invInfo engine %s twin %s; renderer "
              "ReLU decisions replayed %d, twin sign flips %d" % (case, rec.pixels[0].numel(), rays[2], rays[1],
                                                                   eng.info["invInfo"], ref.info["invInfo"],
                                                                   h64.rr.rn.total, h64.rr.rn.flips))
    for k, v in e.items():
        print("[%s] %-20s engine %.2e  fp32 twin %.2e  bar %.0e" % (case, k, v, t32[k], BARS[case].get(k, 0)))
    tie = (rec.tmp_pred.double() - h64.pred)
    ffma = rec.tmp_ffma.double() - h64.pred
    print("[%s] f(TmpVs') over %d vertices, mean |f64| %.2e; minus f64, mean / mean |.| / max |.|: tensor-core "
          "training engine %.2e / %.2e / %.2e, fp32 FFMA engine %.2e / %.2e / %.2e, plain fp32 twin %.2e / %.2e / %.2e"
          % (case, tie.numel(), float(h64.pred.abs().mean()), float(tie.mean()), float(tie.abs().mean()),
             float(tie.abs().max()), float(ffma.mean()), float(ffma.abs().mean()), float(ffma.abs().max()),
             float((h32.pred - h64.pred).mean()), float((h32.pred - h64.pred).abs().mean()),
             float((h32.pred - h64.pred).abs().max())))
    assert counts[-1]["any"] == 0, counts
    print("[%s] extra template points %d, max |twin's own - engine's| %.2e" % (case, rec.extra.shape[0],
                                                                                h64.glue.extra_diff))
    assert h64.glue.extra_diff < 1e-6
    # the engine's sign is replayed; it must be the right one wherever |f| is not within rounding of 0
    assert flip_max < SIGN_BOUND, (case, flip_max)
    assert rec.relu_mismatch == 0
    assert inside > 0 and outside > 0
    assert (dil > 0) == (RADIUS[case] > 0.02)
    if RADIUS[case] > 0.02:
        assert ncov > K     # crowded pixels exist; they are saturated (module docstring), so K truncation is not seen
    assert eng.info["pc_loss"].keys() == ref.info["pc_loss"].keys()
    assert eng.info["rayInfo"] == ref.info["rayInfo"]
    if rays is None:
        assert eng.info["rayInfo"][1] == 0
    else:
        keep, kc, n_conv = rays
        assert kc["any"] <= 0.01 * n_conv, kc
        assert eng.info["rayInfo"][1] == n_conv - kc["any"] > 0
        assert eng.info["invInfo"] == ref.info["invInfo"] and eng.info["invInfo"][0] == eng.info["rayInfo"][1]
        assert len(rec.colors) == 1 and len(h64.rr.colors) == 1
        dc = float((rec.colors[0].double() - h64.rr.colors[0].double()).abs().max())
        print("[%s] max |c_engine - c_twin| %.2e (kink margin %.0e)" % (case, dc, TW.KINK_MARGIN))
        assert dc < TW.KINK_MARGIN
    # the engine run is deterministic
    rec2, eng2 = _engine(case, monkeypatch, move=move, keep=None if rays is None else rays[0])
    assert torch.equal(rec2.tmp[0], rec.tmp[0])
    assert eng2.loss == eng.loss and eng2.info == eng.info and torch.equal(eng2.disp, eng.disp)
    assert (eng.dtmp is None) == (eng2.dtmp is None) and (eng.dtmp is None or torch.equal(eng.dtmp, eng2.dtmp))
    for part in ("direct", "implicit"):
        for name in getattr(eng, part):
            assert torch.equal(getattr(eng, part)[name], getattr(eng2, part)[name]), (case, part, name)
    assert set(e) == set(BARS[case]), (case, sorted(e))
    for k, v in e.items():
        assert v <= BARS[case][k], (case, k, v)


CONTROLS = {"radius +1%": dict(radius_scale=1.01), "dilation +1 pixel": dict(dilate_delta=1),
            "laplacian L^T": dict(mesh_controls=dict(transpose=True)),
            "edge loss over 2E": dict(mesh_controls=dict(half=True)),
            "normal pairs unique": dict(mesh_controls=dict(unique_pairs=True)),
            "normal pairs without -n_j": dict(mesh_controls=dict(same_side=True)), "GM c +1%": dict(c=0.0101),
            "SGD lr +1%": dict(lr_scale=1.01), "inner deformer gradients dropped": dict(drop_inner=True),
            "own |f|": dict(replay_sign=False), "root pose +1e-4 rad": dict(pose_delta=1e-4),
            "PE band weight +1e-3": dict(pe_band_delta=1e-3), "softplus beta +1%": dict(sdf_beta=101.0),
            "renderer PE band weight +1e-3": dict(render_pe_delta=1e-3),
            "no renderer ReLU replay": dict(render_relu=False),
            "Jacobian entry x(1+1e-3)": dict(jac_scale=1.0 + 1e-3), "one mean over all rays": dict(pooled_mean=True)}
CONTROL_CASES = {"mask": ("radius +1%", "dilation +1 pixel", "SGD lr +1%",
                          "inner deformer gradients dropped", "root pose +1e-4 rad", "PE band weight +1e-3",
                          "softplus beta +1%"),
                 "mesh": ("radius +1%", "laplacian L^T", "edge loss over 2E", "normal pairs unique",
                          "normal pairs without -n_j", "SGD lr +1%", "softplus beta +1%"),
                 "defconst": ("radius +1%", "GM c +1%", "SGD lr +1%", "inner deformer gradients dropped",
                              "root pose +1e-4 rad", "PE band weight +1e-3", "softplus beta +1%"),
                 "sdf": ("radius +1%", "own |f|", "softplus beta +1%"),
                 "shipped": ("radius +1%", "dilation +1 pixel", "GM c +1%", "SGD lr +1%",
                             "inner deformer gradients dropped", "own |f|", "root pose +1e-4 rad",
                             "PE band weight +1e-3", "softplus beta +1%"),
                 "step": ("radius +1%", "GM c +1%", "SGD lr +1%", "inner deformer gradients dropped", "own |f|",
                          "root pose +1e-4 rad", "PE band weight +1e-3", "softplus beta +1%",
                          "renderer PE band weight +1e-3", "no renderer ReLU replay", "Jacobian entry x(1+1e-3)",
                          "one mean over all rays")}
# controls that cannot change this scene's figures, and why
MAY_PASS = {"normal pairs unique": "the marching-cubes template is manifold (two faces per edge), where the literal "
                                   "pair comprehension and the unique pairs are the same pair"}
# the bars each control must fail, beyond failing one: together they cover every bar
_GROUPS = ("displacement", "translator", "poses", "trans", "latent")
FAILS = {("mask", "radius +1%"): ("mask_loss",) + _GROUPS, ("mask", "softplus beta +1%"): ("pc_loss_sdf",),
         ("mesh", "radius +1%"): ("mask_loss",), ("mesh", "laplacian L^T"): ("lap_loss", "displacement"),
         ("mesh", "edge loss over 2E"): ("edge_loss", "displacement"),
         ("mesh", "normal pairs without -n_j"): ("norm_loss",), ("mesh", "softplus beta +1%"): ("pc_loss_sdf",),
         ("defconst", "radius +1%"): ("mask_loss",),
         ("defconst", "GM c +1%"): ("defconst_loss", "displacement", "translator", "poses", "latent"),
         ("defconst", "softplus beta +1%"): ("pc_loss_sdf",),
         ("sdf", "radius +1%"): ("mask_loss",), ("sdf", "softplus beta +1%"): ("loss", "pc_loss_sdf"),
         ("sdf", "own |f|"): ("sdf",),
         ("shipped", "radius +1%"): ("loss", "mask_loss", "pc_loss_sdf", "sdf") + _GROUPS,
         ("shipped", "GM c +1%"): ("defconst_loss",),
         ("step", "radius +1%"): ("mask_loss",), ("step", "SGD lr +1%"): ("displacement",),
         ("step", "GM c +1%"): ("defconst_loss", "translator", "poses", "latent"),
         ("step", "inner deformer gradients dropped"): ("trans",), ("step", "own |f|"): ("sdf",),
         ("step", "softplus beta +1%"): ("grad_loss", "pc_loss_sdf"),
         ("step", "Jacobian entry x(1+1e-3)"): ("def_loss",),
         ("step", "renderer PE band weight +1e-3"): ("renderer",),
         ("step", "one mean over all rays"): ("loss", "color_loss", "normal_loss", "TmpPs", "renderer", "implicit sdf",
                                              "implicit translator", "implicit poses", "implicit trans",
                                              "implicit latent")}


@pytest.mark.parametrize("case,control", [(c, k) for c in CASES for k in CONTROL_CASES[c]])
def test_template_negative_controls_fail_their_bars(case, control, monkeypatch):
    rec, eng = _engine_case(case, monkeypatch)[:2]
    bad, hold = _twin(case, rec, torch.float64, monkeypatch, **CONTROLS[control])
    e = _figures(case, eng, bad)
    over = _bar_ratios(case, e)
    print("\n[%s / %s] figure (figure / bar): %s" % (case, control, ", ".join("%s %.2e (%.1f)" % (k, e[k], over[k])
                                                                             for k in e)))
    if control == "no renderer ReLU replay" and hold.rr.rn.flips == 0:
        print("[%s / %s] the replay flipped no renderer decision: nothing to control" % (case, control))
        return
    if control == "own |f|" and hold.sign_flips == 0:
        print("[%s / %s] the replay flipped no sign of the |f| tie: nothing to control" % (case, control))
        return
    if control in MAY_PASS and max(over.values()) <= 1.0:
        print("[%s / %s] %s" % (case, control, MAY_PASS[control]))
        return
    assert max(over.values()) > 1.0, (case, control, e)
    for k in FAILS.get((case, control), ()):
        assert over[k] > 1.0, (case, control, k, e[k])


def test_every_template_bar_has_a_failing_control():
    for case in CASES:
        covered = set(k for (c, _), keys in FAILS.items() if c == case for k in keys)
        assert covered == set(BARS[case]), (case, sorted(set(BARS[case]) - covered))
