"""Float64 twin of one optimisation step (OptimNetwork.forward_rays -> loss.backward() -> propagateTmpPsGrad): the
eikonal, offset, def_regu, colour and weighted-normal terms and the implicit term of propagateTmpPsGrad, taking every
decision from an engine run.  Not collected by pytest: used by test_gpu_train_step_fp64.py.

The scene is test_optim_step_gpu.build()'s (2 frames of 96x96, synth modules).  The engine run is fp32 with the
tensor-core training engine on; test-side wrappers (monkeypatch, no product hooks) record:
  1. the tracer's output: the OptimizeSurfacePs points and convergence mask;
  2. every utils.sample_points draw (eikonal samples, def_regu samples);
  3. the ReLU pattern of every translator and renderer evaluation, read from the activation tiles TcMlpFunction keeps
     for the reverse sweep (train_ops.DEBUG_LAST): the value row of each point (the only row of a ch = 1 launch, row 0
     of a ch = 4 launch), keyed by the module and a hash of the points evaluated (the renderer's `points` argument,
     TmpPs on both sides, not its input row);
  4. for the surface-point branch, the inputs of the decisions that cannot be replayed: the sampler's grid coordinates
     (LBS cell choice), the determinants of every 3x3 matrix inverted (Fast3x3Minv's |det| < 1e-4 test) and the
     rendered colours (the kink of the colour loss's L1 norm).  `keep_mask` turns them into the rays that are removed
     from both runs by AND-ing them out of the recorded convergence mask; a second engine run takes that mask.
The twin is a copy of the SDF, deformer, renderer and SyntheticDataset rebuilt from the same synth seeds, converted to
float64 (or kept fp32 for the fp32 twin), run with the training engine off (torch autograd, create_graph double
backward), with:
  1. the recorded tracer output injected;
  2. the recorded samples injected;
  3. the translator's and the renderer's `relu` replaced by modules that apply the engine's pattern for the points
     being evaluated;
  4. utils.singular_values_3x3 replaced by torch.linalg.svdvals (the plain high-precision reference: the engine keeps
     the device kernel, which is thereby checked inside the step).
The twin's CompositeDeformer reports _fusable() == False, so that compute_deformed_normals(..., 'test') and
propagateTmpPsGrad take their autograd branches, and the fp32 field-engine entry points (ops.sdf_forward,
ops.deform_forward, ops.render_forward, ops.tc_mlp_forward, ops.shade_geometry, train_ops.tc_mlp) raise while it
runs: their fp32 results would otherwise pass unnoticed into the float64 step by type promotion.  The float64 device
kernels the twin does use, the trilinear sampler of GridSamplerMine and Fast3x3Minv, are pinned to float64
restatements by test_gpu_grid_sampler.py and test_gpu_parity.py."""
import collections
import hashlib
import types

import torch

import grid_sampler_ref as GS
import helpers as H

DEV = "cuda"

# half-widths of the decisions keep_mask removes
CELL_MARGIN = 1e-5      # sampler x within this many cells of an integer (cell face, border)
KINK_MARGIN = 1e-3      # |gt - c| of any colour component
DET_MARGIN = 1e-2       # |det| within this fraction of Fast3x3Minv's threshold
DET_THRESHOLD = 1e-4

FP32_ENTRY_POINTS = (("ops", "sdf_forward"), ("ops", "deform_forward"), ("ops", "render_forward"),
                     ("ops", "tc_mlp_forward"), ("ops", "shade_geometry"), ("train_ops", "tc_mlp"))

Step = collections.namedtuple("Step", "loss info direct implicit dtmp")


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


def images(N, Hh, Ww, dtype):
    """The step's colour and normal images: seeded, with about 5 % of the normal pixels zero (invalid)."""
    g = torch.Generator().manual_seed(5)
    img = torch.rand(N, Hh, Ww, 3, generator=g) * 2 - 1
    nrm = torch.nn.functional.normalize(torch.randn(N, Hh, Ww, 3, generator=g), dim=-1)
    nrm[torch.rand(N, Hh, Ww, generator=g) < 0.05] = 0.0
    return img.to(DEV).to(dtype), nrm.to(DEV).to(dtype)


class Record:
    """Decisions of one engine run."""

    def __init__(self):
        self.trace = []        # (points, convergence mask) per OptimizeSurfacePs call
        self.samples = []      # utils.sample_points outputs, in call order
        self.relu = {}         # (module, points_key) -> [layer masks [P, 512] bool]
        self.relu_repeats = 0  # evaluations of points already recorded (a ch = 1 and a ch = 4 launch)
        self.relu_mismatch = 0  # ReLU decisions on which such repeated evaluations disagree
        self.grids = []        # sampler grid coordinates [P,3] fp32, per LBS evaluation
        self.dets = []         # float64 determinants [P] of the matrices of each 3x3 inversion
        self.colors = []       # renderer outputs [P,3]
        self.vol_shape = None  # the skinning volume's shape


def points_key(pts):
    """The points an evaluation sees, as fp32 (the twin's float64 copies of recorded points round back exactly)."""
    return hashlib.sha1(pts.detach().reshape(-1, 3).float().contiguous().cpu().numpy().tobytes()).hexdigest()


def record_engine(monkeypatch, net, rec, surface=False, keep=None):
    """Wrap the engine run's decision points so that `rec` receives them.  surface=False hands forward_rays an
    all-false convergence mask (the surface-point branch is skipped); otherwise the tracer's mask AND `keep`."""
    H.dropin()
    import MCAcc
    import utils
    import model.optim as optim
    from selfreconcode_b200 import _lib, train_ops
    trace0, sample0, mlp0 = utils.OptimizeSurfacePs, utils.sample_points, train_ops.tc_mlp
    sampler0, fdminv0, minv_u0, minv_o0 = (MCAcc.GridSamplerMine3dFunction, utils.FastDiff3x3MinvFunction,
                                           utils.Fast3x3Minv, optim.Fast3x3Minv)
    tr, rn = net.deformer.defs[0], net.netRender
    tr_train0, rn_train0 = tr.forward_train, rn.forward_train
    rec.vol_shape = tuple(net.deformer.defs[1].ws.shape)
    current = []
    tracing = []

    def trace(*a, **k):
        tracing.append(True)
        try:
            p, ok = trace0(*a, **k)
        finally:
            tracing.pop()
        if not surface:
            ok = torch.zeros_like(ok)
        elif keep is not None:
            ok = ok & keep
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

    def rn_train(points, *a, **k):
        current.append(("renderer", points_key(points)))
        try:
            out = rn_train0(points, *a, **k)
        finally:
            current.pop()
        rec.colors.append(out.detach().clone())
        return out

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

    def dets(m):
        if not tracing:
            rec.dets.append(torch.linalg.det(m.detach().double()))

    class Sampler:
        @staticmethod
        def apply(vol, grid):
            if not tracing:
                rec.grids.append(grid.detach().reshape(-1, 3).clone())
            return sampler0.apply(vol, grid)

    class FastDiffMinv:
        @staticmethod
        def apply(m):
            dets(m)
            return fdminv0.apply(m)

    def minv(f0):
        def f(m):
            dets(m)
            return f0(m)
        return f

    monkeypatch.setattr(utils, "OptimizeSurfacePs", trace)
    monkeypatch.setattr(utils, "sample_points", sample)
    monkeypatch.setattr(train_ops, "tc_mlp", mlp)
    monkeypatch.setattr(tr, "forward_train", tr_train)
    monkeypatch.setattr(rn, "forward_train", rn_train)
    monkeypatch.setattr(MCAcc, "GridSamplerMine3dFunction", Sampler)
    monkeypatch.setattr(utils, "FastDiff3x3MinvFunction", FastDiffMinv)
    monkeypatch.setattr(utils, "Fast3x3Minv", minv(minv_u0))
    monkeypatch.setattr(optim, "Fast3x3Minv", minv(minv_o0))


def keep_mask(rec, gt):
    """Rays whose step takes a decision the twin cannot replay, from a first engine run `rec` over all converged rays;
    gt [rays, 3] the colour image at every ray.  -> (keep [rays] bool, {reason: rays excluded}, converged rays).
    Reasons: the sampler's x (the kernel's own rule, grid_sampler_ref.unnormalise) within CELL_MARGIN cells of a cell
    face or the volume's border, where the corner choice or the border mask changes; any |gt - c| < KINK_MARGIN, the
    kink of the colour loss's |.|; |det| within DET_MARGIN of Fast3x3Minv's threshold, for the deformer Jacobian
    (cardinal rays, normal weights) and b^T b (propagateTmpPsGrad)."""
    ok = rec.trace[0][1]
    idx = ok.nonzero().squeeze(1)
    n = idx.numel()
    D, Hv, W = rec.vol_shape[-3:]
    cell = torch.zeros(n, dtype=torch.bool, device=ok.device)
    for g in rec.grids:
        if g.shape[0] != n:
            continue
        for k, size in enumerate((W, Hv, D)):
            x = GS.unnormalise(g[:, k].contiguous(), size).double()
            cell |= ((x - x.round()).abs() < CELL_MARGIN) & (x > -1) & (x < size)
    det = torch.zeros_like(cell)
    for d in rec.dets:
        if d.numel() == n:
            det |= (d.abs() - DET_THRESHOLD).abs() < DET_MARGIN * DET_THRESHOLD
    kink = torch.zeros_like(cell)
    g = gt[idx].double()
    for c in rec.colors:
        if c.shape[0] == n:
            kink |= ((g - c.double()).abs() < KINK_MARGIN).any(1)
    keep = torch.ones_like(ok)
    keep[idx[cell | det | kink]] = False
    counts = {"LBS cell face": int(cell.sum()), "colour L1 kink": int(kink.sum()), "3x3 inverse threshold":
              int(det.sum()), "any": int((cell | det | kink).sum())}
    return keep, counts, n


class ReplayReLU(torch.nn.Module):
    """relu(x) with the engine's pattern: x * mask.  `key` is set by the module's forward to (module, points_key) of
    the points it evaluates and `layer` counts its hidden layers.  Counts where the twin's own sign disagrees with the
    engine's decision (flips) and the decisions it replays.  apply=False counts the same but returns the twin's own
    relu(x)."""

    def __init__(self, masks, apply=True):
        super().__init__()
        self.masks = masks
        self.apply_masks = apply
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
        if not self.apply_masks:
            return torch.relu(x)
        return x * m.to(x.dtype)


def _refuse(name):
    def f(*a, **k):
        raise RuntimeError("the float64 twin reached the fp32 field-engine entry point %s" % name)
    return f


def replay_twin(monkeypatch, net, rec, dtype, relu=True, render_relu=True, pe_band_delta=0.0, render_pe_delta=0.0,
                sdf_beta=None, pose_delta=0.0, jac_scale=1.0, pooled_mean=False):
    """Wrap the twin's decision points with the engine's recorded ones and refuse the fp32 entry points.  -> namespace
    of the translator's and the renderer's ReplayReLU (or None) and the colours the twin renders."""
    H.dropin()
    import utils
    from selfreconcode_b200 import ops, train_ops
    mods = {"ops": ops, "train_ops": train_ops}
    for mod, name in FP32_ENTRY_POINTS:
        monkeypatch.setattr(mods[mod], name, _refuse(name))
    monkeypatch.setattr(net.deformer, "_fusable", lambda: False)
    trace = list(rec.trace)
    samples = list(rec.samples)
    monkeypatch.setattr(utils, "OptimizeSurfacePs",
                        lambda *a, **k: (lambda t: (t[0].to(dtype).clone(), t[1].clone()))(trace.pop(0)))
    monkeypatch.setattr(utils, "sample_points", lambda *a, **k: samples.pop(0).to(dtype).clone())
    monkeypatch.setattr(utils, "singular_values_3x3",
                        lambda J: torch.linalg.svdvals(J.double()).to(dtype))
    if pe_band_delta or render_pe_delta:
        # negative controls: the last active band's annealing weight of the translator (deformerRatio) or of the
        # renderer's view direction (its multires_v) moved
        aw0 = ops.annealing_weights
        multires_v = net.netRender.multires_v

        def aw(multires, ratio):
            w = list(aw0(multires, ratio))      # one weight per band
            delta = pe_band_delta if ratio == H.RATIO["deformerRatio"] else \
                render_pe_delta if multires == multires_v else 0.0
            if delta:
                w[max(i for i in range(len(w)) if w[i] > 0)] += delta
            return w
        monkeypatch.setattr(ops, "annealing_weights", aw)
    if sdf_beta is not None:
        # negative control: the SDF's softplus sharpness
        net.sdf.softplus = torch.nn.Softplus(beta=sdf_beta)
    if pose_delta:
        # negative control: one axis-angle component of the root joint, every frame
        with torch.no_grad():
            net.dataset.poses.view(net.dataset.poses.shape[0], 24, 3)[:, 0, 1] += pose_delta
    if pooled_mean:
        # negative control: the colour and normal losses as one mean over all rays instead of the mean of per-frame means
        import model.optim as optim
        monkeypatch.setattr(optim, "_scatter_mean",
                            lambda src, index, n: src.mean(0, keepdim=True).expand((n,) + tuple(src.shape[1:])))
    if jac_scale != 1.0:
        # negative control: entry (0, 0) of every deformer Jacobian the twin takes by autograd
        cj0 = utils.compute_Jacobian

        def cj(*a, **k):
            J = cj0(*a, **k)
            s = torch.ones(3, 3, dtype=J.dtype, device=J.device)
            s[0, 0] = jac_scale
            return J * s
        monkeypatch.setattr(utils, "compute_Jacobian", cj)
    out = types.SimpleNamespace(tr=None, rn=None, colors=[])
    if relu:
        out.tr = ReplayReLU(rec.relu)
        tr = net.deformer.defs[0]
        tr.relu = out.tr
        fwd0 = tr.forward

        def fwd(ps, *a, **k):
            out.tr.key, out.tr.layer = ("translator", points_key(ps)), 0
            return fwd0(ps, *a, **k)
        monkeypatch.setattr(tr, "forward", fwd)
    rn = net.netRender
    rfwd0 = rn.forward
    if any(k[0] == "renderer" for k in rec.relu):
        out.rn = ReplayReLU(rec.relu, apply=render_relu)
        rn.relu = out.rn

    def rfwd(points, *a, **k):
        if out.rn is not None:
            out.rn.key, out.rn.layer = ("renderer", points_key(points)), 0
        c = rfwd0(points, *a, **k)
        out.colors.append(c.detach().clone())
        return c
    monkeypatch.setattr(rn, "forward", rfwd)
    return out


def run_step(net, data, rays, fids, conf, dtype, engine):
    """forward_rays -> backward -> propagateTmpPsGrad.  -> Step(loss, info (with invInfo), parameter gradients per
    group after backward (direct) and of propagateTmpPsGrad alone (implicit), dL/dTmpPs or None)."""
    from selfreconcode_b200 import train_ops
    flag = train_ops.TC_TRAIN_ENABLED
    train_ops.TC_TRAIN_ENABLED = engine
    try:
        net.conf = conf
        ps = [p for g in groups(net, data).values() for p in g]
        for p in ps:
            p.grad = None
        img, nrm = images(fids.numel(), data.H, data.W, dtype)
        bi, ri, ci = rays["batch_inds"].to(DEV), rays["rows"].to(DEV), rays["cols"].to(DEV)
        with torch.random.fork_rng(devices=[torch.device(DEV)]):
            torch.manual_seed(9)
            loss = net.forward_rays({"img": img, "normal": nrm}, bi, ri, ci,
                                    rays["init_pts"].to(DEV).to(dtype).clone(), H.RATIO, fids)
        loss.backward()
        info = dict(net.info)
        direct = flat_grads(net, data)
        dtmp = None if net.TmpPs is None or net.TmpPs.grad is None else net.TmpPs.grad.detach().double().clone()
        for p in ps:
            p.grad = None
        net.propagateTmpPsGrad(fids, H.RATIO)
        info["invInfo"] = net.info["invInfo"]
        return Step(loss.item(), info, direct, flat_grads(net, data), dtmp)
    finally:
        train_ops.TC_TRAIN_ENABLED = flag
