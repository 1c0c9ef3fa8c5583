"""Float64 twin of the regulariser half (eikonal, offset, def_regu) of one optimisation step (OptimNetwork.forward_rays
-> loss.backward() -> propagateTmpPsGrad) that takes every decision from an engine run.  Not collected by pytest: used by
test_gpu_train_step_fp64.py.

The scene is test_optim_step_gpu.build()'s (2 frames of 96x96, synth modules).  The engine run is fp32 with the
tensor-core training engine on; test-side wrappers (monkeypatch, no product hooks) record:
  1. the tracer's output: the OptimizeSurfacePs points and convergence mask;
  2. every utils.sample_points draw (eikonal samples, def_regu samples);
  3. the ReLU pattern of every translator evaluation, read from the activation tiles TcMlpFunction keeps for the
     reverse sweep (train_ops.DEBUG_LAST): the value row of each point (the only row of a ch = 1 launch, row 0 of a
     ch = 4 launch), keyed by the module and a hash of the points evaluated.
The twin is a copy of the SDF, deformer, renderer and SyntheticDataset rebuilt from the same synth seeds, converted to
float64 (or kept fp32 for the fp32 twin), run with the training engine off (torch autograd, create_graph double
backward), with:
  1. the recorded tracer output injected;
  2. the recorded samples injected;
  3. the translator's `relu` replaced by a module that applies the engine's pattern for the points being evaluated;
  4. utils.singular_values_3x3 replaced by torch.linalg.svdvals (the plain high-precision reference: the engine keeps
     the device kernel, which is thereby checked inside the step).
The surface-point branch (colour, normal and implicit terms) is switched off in both runs by injecting an all-false
convergence mask: the terms here depend on the traced points only as the base of the samples."""
import hashlib
import types

import torch

import helpers as H

DEV = "cuda"


def groups(net, data):
    """parameter group name -> list of parameters, in a fixed order."""
    return {"sdf": list(net.sdf.parameters()), "translator": list(net.deformer.defs[0].parameters()),
            "renderer": list(net.netRender.parameters()), "poses": [data.poses], "trans": [data.trans],
            "latent": list(data.conds.parameters())}


def flat_grads(net, data):
    out = {}
    for name, ps in groups(net, data).items():
        gs = [p.grad.detach().double().reshape(-1) if p.grad is not None else torch.zeros(p.numel(), dtype=torch.float64,
                                                                                          device=DEV)
              for p in ps if p.requires_grad]
        out[name] = torch.cat(gs) if gs else torch.zeros(0, dtype=torch.float64, device=DEV)
    return out


def make_twin(dtype, n_frames=2, Hh=96, Ww=96):
    """(OptimNetwork, dataset) rebuilt from the seeds test_optim_step_gpu.build() uses, in `dtype`."""
    H.dropin()
    from selfreconcode_b200 import synth
    from model.Deformer import CompositeDeformer
    from model.optim import OptimNetwork
    from model.CameraMine import RectifiedPerspectiveCameras
    sdf = synth.make_sdf().to(dtype).to(DEV)
    comp = CompositeDeformer([synth.make_translator(), synth.make_skinner(resolution=(33, 57, 17))]).to(dtype).to(DEV)
    rn = synth.make_render().to(dtype).to(DEV)
    data = synth.SyntheticDataset(n_frames, Hh, Ww).to(dtype).to(DEV)
    f, pp, R, T, _, _ = data.get_camera_parameters(n_frames, DEV)
    cams = RectifiedPerspectiveCameras(f.detach(), pp.detach(), R, T.detach(), image_size=[(Ww, Hh)])
    holder = types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=cams))
    net = OptimNetwork(sdf, comp, None, holder, rn)
    net.dataset = data
    return net, data


class Record:
    """Decisions of one engine run."""

    def __init__(self):
        self.trace = []        # (points, convergence mask) per OptimizeSurfacePs call
        self.samples = []      # utils.sample_points outputs, in call order
        self.relu = {}         # (module, points_key) -> [layer masks [P, 512] bool]
        self.relu_repeats = 0  # evaluations of points already recorded (a ch = 1 and a ch = 4 launch)
        self.relu_mismatch = 0  # ReLU decisions on which such repeated evaluations disagree


def points_key(pts):
    """The points an evaluation sees, as fp32 (the twin's float64 copies of recorded points round back exactly)."""
    return hashlib.sha1(pts.detach().reshape(-1, 3).float().contiguous().cpu().numpy().tobytes()).hexdigest()


def record_engine(monkeypatch, net, rec, surface=False):
    """Wrap the engine run's decision points so that `rec` receives them.  surface=False hands forward_rays an
    all-false convergence mask (the surface-point branch is skipped)."""
    H.dropin()
    import utils
    from selfreconcode_b200 import _lib, train_ops
    trace0, sample0, mlp0 = utils.OptimizeSurfacePs, utils.sample_points, train_ops.tc_mlp
    tr = net.deformer.defs[0]
    tr_train0 = tr.forward_train
    current = []

    def trace(*a, **k):
        p, ok = trace0(*a, **k)
        if not surface:
            ok = torch.zeros_like(ok)
        rec.trace.append((p.detach().clone(), ok.clone()))
        return p, ok

    def sample(*a, **k):
        out = sample0(*a, **k)
        rec.samples.append(out.detach().clone())
        return out

    def tr_train(pts, *a, **k):
        current.append(("translator", points_key(pts)))
        try:
            return tr_train0(pts, *a, **k)
        finally:
            current.pop()

    def mlp(x0, cfg, weights, biases):
        if _lib.SR_ACT_RELU not in cfg.acts or not current:
            return mlp0(x0, cfg, weights, biases)
        train_ops.DEBUG_LAST = {}
        try:
            out = mlp0(x0, cfg, weights, biases)
            d = train_ops.DEBUG_LAST
            P = d["M"] // cfg.ch
            masks = []
            for i, tiles in enumerate(d["acts"]):
                a = train_ops.unpack_tiles(tiles, d["M"], d["kpads"][i + 1])
                masks.append(a.view(P, cfg.ch, -1)[:, 0, :d["widths"][i]] > 0)
            key = current[-1]
            if key in rec.relu:
                rec.relu_repeats += 1
                rec.relu_mismatch += sum(int((a != b).sum()) for a, b in zip(rec.relu[key], masks))
            else:
                rec.relu[key] = masks
        finally:
            train_ops.DEBUG_LAST = None
        return out

    monkeypatch.setattr(utils, "OptimizeSurfacePs", trace)
    monkeypatch.setattr(utils, "sample_points", sample)
    monkeypatch.setattr(train_ops, "tc_mlp", mlp)
    monkeypatch.setattr(tr, "forward_train", tr_train)


class ReplayReLU(torch.nn.Module):
    """relu(x) with the engine's pattern: x * mask.  `key` is set by the module's forward to (module, points_key) of
    the points it evaluates and `layer` counts its hidden layers.  Counts where the twin's own sign disagrees with the
    engine's decision (flips) and the decisions it replays."""

    def __init__(self, masks):
        super().__init__()
        self.masks = masks
        self.key = None
        self.layer = 0
        self.flips = 0
        self.total = 0

    def forward(self, x):
        assert self.key in self.masks, "no engine ReLU pattern for these points"
        m = self.masks[self.key][self.layer]
        self.layer += 1
        assert m.shape == x.shape, (m.shape, x.shape)
        with torch.no_grad():
            self.flips += int(((x > 0) != m).sum())
            self.total += m.numel()
        return x * m.to(x.dtype)


def replay_twin(monkeypatch, net, rec, dtype, relu=True, pe_band_delta=0.0, sdf_beta=None):
    """Wrap the twin's decision points with the engine's recorded ones.  -> the ReplayReLU module (or None)."""
    H.dropin()
    import utils
    from selfreconcode_b200 import ops
    trace = list(rec.trace)
    samples = list(rec.samples)
    monkeypatch.setattr(utils, "OptimizeSurfacePs",
                        lambda *a, **k: (lambda t: (t[0].to(dtype).clone(), t[1].clone()))(trace.pop(0)))
    monkeypatch.setattr(utils, "sample_points", lambda *a, **k: samples.pop(0).to(dtype).clone())
    monkeypatch.setattr(utils, "singular_values_3x3",
                        lambda J: torch.linalg.svdvals(J.double()).to(dtype))
    if pe_band_delta:
        # negative control: the last active band's annealing weight of the translator moved by pe_band_delta
        aw0 = ops.annealing_weights

        def aw(multires, ratio):
            w = list(aw0(multires, ratio))      # one weight per band
            if ratio == H.RATIO["deformerRatio"]:
                w[max(i for i in range(len(w)) if w[i] > 0)] += pe_band_delta
            return w
        monkeypatch.setattr(ops, "annealing_weights", aw)
    if sdf_beta is not None:
        # negative control: the SDF's softplus sharpness
        net.sdf.softplus = torch.nn.Softplus(beta=sdf_beta)
    rr = None
    if relu:
        rr = ReplayReLU(rec.relu)
        tr = net.deformer.defs[0]
        tr.relu = rr
        fwd0 = tr.forward

        def fwd(ps, *a, **k):
            rr.key, rr.layer = ("translator", points_key(ps)), 0
            return fwd0(ps, *a, **k)
        monkeypatch.setattr(tr, "forward", fwd)
    return rr


def run_step(net, data, rays, fids, conf, dtype, engine):
    """forward_rays -> backward -> propagateTmpPsGrad.  -> (loss, info, grads per group)."""
    from selfreconcode_b200 import train_ops
    flag = train_ops.TC_TRAIN_ENABLED
    train_ops.TC_TRAIN_ENABLED = engine
    try:
        net.conf = conf
        for ps in groups(net, data).values():
            for p in ps:
                p.grad = None
        g = torch.Generator().manual_seed(5)
        N, Hh, Ww = fids.numel(), data.H, data.W
        img = (torch.rand(N, Hh, Ww, 3, generator=g) * 2 - 1).to(DEV).to(dtype)
        bi, ri, ci = rays["batch_inds"].to(DEV), rays["rows"].to(DEV), rays["cols"].to(DEV)
        with torch.random.fork_rng(devices=[torch.device(DEV)]):
            torch.manual_seed(9)
            loss = net.forward_rays({"img": img}, bi, ri, ci, rays["init_pts"].to(DEV).to(dtype).clone(), H.RATIO,
                                    fids)
        info = dict(net.info)
        loss.backward()
        net.propagateTmpPsGrad(fids, H.RATIO)
        return loss.item(), info, flat_grads(net, data)
    finally:
        train_ops.TC_TRAIN_ENABLED = flag
