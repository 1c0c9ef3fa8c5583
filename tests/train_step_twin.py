"""Float64 twin of one optimisation step (OptimNetwork.forward_rays -> loss.backward() -> propagateTmpPsGrad): the
eikonal, offset, def_regu, colour and weighted-normal terms and the implicit term of propagateTmpPsGrad, taking every
decision from an engine run; and of forward()'s template term (record_template / replay_template, below): the point
silhouette, mesh regularisers, def_consistent term, inner SGD step on TmpVs and the |f| tie.  Not collected by pytest:
used by test_gpu_train_step_fp64.py and test_gpu_train_template_fp64.py.

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
propagateTmpPsGrad take their autograd branches, and the fp32 entry points (ops.sdf_forward, ops.deform_forward,
ops.render_forward, ops.tc_mlp_forward, ops.shade_geometry, train_ops.tc_mlp, ops.points_silhouette,
ops.mesh_regularizers, ops.sdf_refine_band) raise while it runs: their fp32 results would otherwise pass unnoticed
into the float64 step by type promotion.  The float64 device kernels the twin does use, the trilinear sampler of
GridSamplerMine and Fast3x3Minv, are pinned to float64 restatements by test_gpu_grid_sampler.py and test_gpu_parity.py.

For the template term the engine run also records the marching-cubes template, the mesh seed, the point silhouette's
fp32 screen points, dL/dTmpVs at the inner SGD step and the fp32 values the |f| tie's sign is taken on; the twin
replays the template and the seed, renders with Silhouette64 (points_silhouette_ref in float64, projected by
raster.screen_vertices in the twin's dtype), takes mesh_reg_ref's regularisers and applies the engine's sign to its own
f(TmpVs').  Every template vertex feeds every figure, so the vertices within a decision the twin cannot replay
(template_borderline) are moved by MOVE_STEP in a further engine run instead of being dropped.  forward()'s glue
between the two terms (the gt-mask selection of the seed pixels, the sample_pix subsampling and the draw of the extra
template points for the eikonal and def_regu samples) is restated by forward_glue and checked on both sides."""
import collections
import hashlib
import types

import numpy as np
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
                     ("ops", "tc_mlp_forward"), ("ops", "shade_geometry"), ("train_ops", "tc_mlp"),
                     ("ops", "points_silhouette"), ("ops", "mesh_regularizers"), ("ops", "sdf_refine_band"))

# half-widths of the template decisions template_borderline finds
SIL_REL = 1e-4          # |d2 - r^2| within this fraction of r^2 at some pixel (point coverage)
Z_TIE = 1e-6            # depth within this fraction of the K-th kept point's depth at a pixel with more than K
MOVE_STEP = 2e-4        # what the wrapped discretizeSDF adds to each coordinate of a borderline vertex

Step = collections.namedtuple("Step", "loss info direct implicit dtmp")
TStep = collections.namedtuple("TStep", "loss info direct implicit dtmp disp")


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


def make_twin(dtype, n_frames=2, Hh=96, Ww=96, mesh_raster=False):
    """(OptimNetwork, dataset) rebuilt from the seeds test_optim_step_gpu.build() uses, in `dtype`.  mesh_raster: the
    built-in mesh rasteriser as maskRender, so that a hierarchy level installs the built-in point renderer (forward();
    the twin replays the rasteriser's seed and replaces the point renderer, replay_template)."""
    H.dropin()
    from selfreconcode_b200 import synth
    from model.Deformer import CompositeDeformer
    from model.optim import OptimNetwork
    from model.CameraMine import RectifiedPerspectiveCameras
    from model.raster import MeshRasterizer, RasterSettings, SilhouetteRenderer
    sdf = synth.make_sdf().to(dtype).to(DEV)
    comp = CompositeDeformer([synth.make_translator(), synth.make_skinner(resolution=(33, 57, 17))]).to(dtype).to(DEV)
    rn = synth.make_render().to(dtype).to(DEV)
    data = synth.SyntheticDataset(n_frames, Hh, Ww).to(dtype).to(DEV)
    f, pp, R, T, _, _ = data.get_camera_parameters(n_frames, DEV)
    cams = RectifiedPerspectiveCameras(f.detach(), pp.detach(), R, T.detach(), image_size=[(Ww, Hh)])
    if mesh_raster:
        holder = SilhouetteRenderer(MeshRasterizer(cams, RasterSettings((Hh, Ww))))
    else:
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
        # the template term of forward() (record_template)
        self.tmp = None        # (TmpVs, Tmpfs) as discretizeSDF returned them (borderline vertices moved)
        self.moved = 0         # vertices the wrapped discretizeSDF moved
        self.seed = None       # _mesh_seed's (batch, row, col, start points, front faces)
        self.sil = []          # (fp32 screen points [N,V,3], H, W, fp32 radius, K) per point-silhouette launch
        self.tmp_f32 = None    # the fp32 values the sign of the |f| tie is taken on
        self.tmp_ffma = None   # f(TmpVs') on the fp32 FFMA engine (diagnostic)
        self.tmp_grids = []    # the sampler grids of the template's LBS evaluations (deformed, def_consistent)
        self.pixels = None     # (batch, row, col) forward() hands forward_rays
        self.extra = None      # the extra template points forward() hands forward_rays
        self.tmp_pred = None   # the differentiable tensor-core f(TmpVs') the tie multiplies by that sign


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


# ---- the template term of OptimNetwork.forward (computeTmpPcLoss) -----------------------------------------------------
class Silhouette64(torch.autograd.Function):
    """points_silhouette_ref's soft point silhouette as an autograd function of the screen points [N,V,3] =
    (col, row, Z): float64 on the host, returned in the points' dtype.  K None composites every covering point."""

    @staticmethod
    def forward(ctx, pts, Hh, Ww, r, K):
        import points_silhouette_ref as PS
        ndc = PS.screen_to_ndc(pts.detach().double().cpu().numpy(), Hh, Ww)
        ctx.args = (ndc, Hh, Ww, r, K)
        return torch.from_numpy(PS.silhouette(ndc, Hh, Ww, r, K)).to(pts.device).to(pts.dtype)[..., None]

    @staticmethod
    def backward(ctx, g):
        import points_silhouette_ref as PS
        ndc, Hh, Ww, r, K = ctx.args
        gn = PS.silhouette_grad(ndc, Hh, Ww, r, K, g[..., 0].detach().double().cpu().numpy())
        return torch.from_numpy(PS.ndc_grad_to_screen(gn, Hh, Ww)).to(g.device).to(g.dtype), None, None, None, None


class SilhouetteRenderer64:
    """Stands in for raster.PointsSilhouetteRenderer (OptimNetwork's `takes_tensors` protocol): projects with
    raster.screen_vertices in the vertices' dtype, so autograd reaches the vertices and the cameras' inputs, and
    renders with Silhouette64 at the kernel's fp32 radius.  `radius` is what forward() reads for the gt mask's
    dilation.  Negative controls: radius_scale (the silhouette's radius only), truncate=False (no K truncation),
    dilate_delta (the dilation's radius in pixels)."""
    takes_tensors = True

    def __init__(self, builtin, radius_scale=1.0, truncate=True, dilate_delta=0):
        s = builtin.rasterizer.raster_settings
        self.rasterizer = builtin.rasterizer
        self.radius = s.radius
        if dilate_delta:
            Hh, Ww = s.image_size
            px = int(round(s.radius / 2. * float(min(Hh, Ww)) / 1.2)) + dilate_delta
            self.radius = px * 2. * 1.2 / float(min(Hh, Ww))
        self.r = float(np.float32(s.radius)) * radius_scale
        self.K = s.points_per_pixel if truncate else None

    def __call__(self, verts):
        from model.raster import screen_vertices
        s = self.rasterizer.raster_settings
        return Silhouette64.apply(screen_vertices(verts, self.rasterizer.cameras), s.image_size[0], s.image_size[1],
                                  self.r, self.K)


def _wrap_inner_step(monkeypatch, net, hold, lr_scale=1.0, drop=None):
    """Wrap computeTmpPcLoss so that its TmpOptimizer.step() leaves on `hold`: the gradient on TmpVs (float64), the
    learning rate, and `stepped` = True until computeTmpPcLoss returns; `hold.arm` is then set to hold.replay_sign.
    Negative controls: lr_scale (SGD's learning rate), drop() -> parameters whose .grad is dropped before the step
    (the inner backward's deformer gradients)."""
    pc0 = net.computeTmpPcLoss

    def pc(*a, **k):
        opt = net.TmpOptimizer
        step0 = opt.step

        def step(*sa, **sk):
            g = opt.param_groups[0]
            g["lr"] *= lr_scale
            hold.tmp_grad = net.TmpVs.grad.detach().double().clone()
            hold.lr = g["lr"]
            if drop is not None:
                for p in drop():
                    p.grad = None
            out = step0(*sa, **sk)
            hold.stepped = True
            hold.arm = getattr(hold, "replay_sign", False)
            return out
        opt.step = step
        try:
            return pc0(*a, **k)
        finally:
            opt.step = step0
            hold.stepped = False
    monkeypatch.setattr(net, "computeTmpPcLoss", pc)


def record_template(monkeypatch, net, rec, move=None):
    """Wrap the template term's decision points of an engine run (with record_engine): discretizeSDF (vertex i is
    moved by move[i] * MOVE_STEP on every coordinate, `move` [V] int), _mesh_seed, the point silhouette's fp32
    screen points, TmpVs's gradient at the inner SGD step, the fp32 values the |f| tie takes its sign on and the
    tensor-core values it multiplies (tmp_pred).  The translator's ReLU pattern is record_engine's, and so are the LBS
    grid coordinates; those of the template's two LBS evaluations (_deform in forward(), the def_consistent skinning in
    computeTmpPcLoss) are also listed in rec.tmp_grids.  -> the namespace the step writes (tmp_grad, lr)."""
    H.dropin()
    from selfreconcode_b200 import ops
    disc0, seed0, sil0, ff0 = net.discretizeSDF, net._mesh_seed, ops.points_silhouette, net.sdf.forward_fused
    sdfv0, deform0, pc0 = net._sdf_value, net._deform, net.computeTmpPcLoss
    hold = types.SimpleNamespace(stepped=False, tmp_grad=None, lr=None)

    def grids_of(f0):
        def f(*a, **k):
            start = len(rec.grids)
            out = f0(*a, **k)
            rec.tmp_grids += rec.grids[start:]
            return out
        return f

    def disc(*a, **k):
        v, f = disc0(*a, **k)
        v = v.detach().clone()
        if move is not None:
            assert move.shape[0] == v.shape[0]
            v += MOVE_STEP * move.view(-1, 1).to(v.dtype)
            rec.moved = int((move > 0).sum())
        rec.tmp = (v.clone(), f.clone())
        return v, f

    def seed(*a, **k):
        out = seed0(*a, **k)
        rec.seed = tuple(x.detach().clone() if torch.is_tensor(x) else x for x in out)
        return out

    def sil(pts, Hh, Ww, r, K):
        rec.sil.append((pts.detach().clone(), Hh, Ww, float(np.float32(r)), K))
        return sil0(pts, Hh, Ww, r, K)

    def ff(*a, **k):
        out = ff0(*a, **k)
        if hold.stepped and "refine_about" in k:
            rec.tmp_f32 = out[0].detach().clone()
            # the same points on the fp32 FFMA engine alone (a want_grad evaluation never takes the tensor cores)
            rec.tmp_ffma = ff0(a[0], a[1], True, False)[0].detach().reshape(-1).clone()
        return out

    def sdf_value(pts, ratio):
        p = sdfv0(pts, ratio)
        if hold.stepped:
            rec.tmp_pred = p.detach().reshape(-1).clone()
        return p

    monkeypatch.setattr(net, "discretizeSDF", disc)
    monkeypatch.setattr(net, "_mesh_seed", seed)
    monkeypatch.setattr(net, "_sdf_value", sdf_value)
    monkeypatch.setattr(net, "_deform", grids_of(deform0))
    monkeypatch.setattr(net, "computeTmpPcLoss", grids_of(pc0))
    monkeypatch.setattr(ops, "points_silhouette", sil)
    monkeypatch.setattr(net.sdf, "forward_fused", ff)
    _wrap_inner_step(monkeypatch, net, hold)
    return hold


def depth_near_ties(ndc, Hh, Ww, r, K, rel=Z_TIE):
    """[N,V] bool: points whose depth is within rel of that of the K-th kept point of a pixel with more than K
    covering points (other than being that point): the K truncation may keep the other one on the other side."""
    import points_silhouette_ref as PS
    N, V = ndc.shape[0], ndc.shape[1]
    out = np.zeros((N, V), bool)
    R = PS.rasterize(ndc, Hh, Ww, r, None)
    crowded = R["n_cover"][R["pix"]] > K
    kth = crowded & (R["slot"] == K - 1)
    zk = np.full(N * Hh * Ww, np.nan)
    zk[R["pix"][kth]] = R["z"][kth]
    z = zk[R["pix"]]
    tie = crowded & (np.abs(R["z"] - z) <= rel * np.abs(z)) & (R["slot"] != K - 1)
    out[R["n"][tie], R["p"][tie]] = True
    return out


def template_borderline(rec):
    """Template vertices whose term takes a decision the twin cannot replay, from an engine run `rec`:
    -> ([V] bool, {reason: vertices}).  Reasons: an LBS sampler x (both template evaluations: the deformed template
    and the def_consistent one at TmpVs) within CELL_MARGIN cells of a cell face or the volume's border; a point
    within SIL_REL of covering a pixel (|d2 - r^2|), or within Z_TIE of the depth of a pixel's K-th kept point
    (points_silhouette_ref.borderline_points and depth_near_ties on the engine's own fp32 screen points).  Neither the
    def_consistent term (GMRobustError at c > 0: a rational function, no kink) nor the |f| tie (the engine's sign is
    replayed) takes another decision."""
    import points_silhouette_ref as PS
    V = rec.tmp[0].shape[0]
    N = rec.sil[0][0].shape[0]
    D, Hv, W = rec.vol_shape[-3:]
    cell = torch.zeros(V, dtype=torch.bool, device=DEV)
    assert 1 <= len(rec.tmp_grids) <= 2, len(rec.tmp_grids)
    for g in rec.tmp_grids:
        assert g.shape[0] == N * V, (g.shape, N, V)
        for k, size in enumerate((W, Hv, D)):
            x = GS.unnormalise(g[:, k].contiguous(), size).double()
            near = ((x - x.round()).abs() < CELL_MARGIN) & (x > -1) & (x < size)
            cell |= near.view(-1, V).any(0)
    sil = torch.zeros_like(cell)
    for pts, Hh, Ww, r, K in rec.sil:
        ndc = PS.screen_to_ndc(pts.double().cpu().numpy(), Hh, Ww)
        b = PS.borderline_points(ndc, Hh, Ww, r, K, rel=SIL_REL) | depth_near_ties(ndc, Hh, Ww, r, K)
        sil |= torch.from_numpy(b.any(0)).to(DEV)
    counts = {"LBS cell face": int(cell.sum()), "point silhouette": int(sil.sum()), "any": int((cell | sil).sum())}
    return cell | sil, counts


def replay_template(monkeypatch, net, rec, dtype, radius_scale=1.0, truncate=True, dilate_delta=0, lr_scale=1.0,
                    drop_inner=False, replay_sign=True, mesh_controls=None):
    """The template term's replay in the twin (after replay_twin): discretizeSDF returns the recorded template in
    `dtype` and installs SilhouetteRenderer64 in place of the point renderer update_hierarchical_config has just built;
    the recorded mesh seed; mesh_reg_ref.regularizers in float64 for the device mesh regularisers; the engine's sign
    applied to the twin's f(TmpVs') in the |f| tie: utils.train_fused answers True once, at the tie, _sdf_value stays
    on the twin's module and sdf.forward_fused returns the recorded fp32 values.  Negative controls: radius_scale,
    truncate, dilate_delta (SilhouetteRenderer64), lr_scale, drop_inner (the translator's, poses', translations' and
    latent codes' gradients of the inner backward dropped before the step), replay_sign=False (the twin's own |f|),
    mesh_controls (mesh_reg_ref's switches, and same_side: the normal term without the minus sign of -n_j).
    -> namespace: sign_flips (where the twin's own sign differs from the engine's), flip_f64 (the twin's |f| there),
    sign_total, pred (the twin's f(TmpVs')), tmp_grad, lr."""
    H.dropin()
    import utils
    import mesh_reg_ref as MR
    from selfreconcode_b200 import ops
    data = net.dataset
    hold = types.SimpleNamespace(stepped=False, arm=False, replay_sign=replay_sign, tmp_grad=None, lr=None,
                                 sign_flips=None, flip_f64=None, sign_total=0, pred=None)
    V, F = rec.tmp
    bi, ri, ci, ps, ffi = rec.seed

    def disc(*a, **k):
        net.pcRender = SilhouetteRenderer64(net.pcRender, radius_scale, truncate, dilate_delta)
        return V.to(dtype).clone(), F.clone()

    controls = dict(mesh_controls or {})
    same_side = controls.pop("same_side", False)

    def regs(verts, topo):
        faces, nv = topo
        assert nv == verts.shape[0]
        r = MR.regularizers(verts.double().cpu(), faces.cpu(), **controls)
        if same_side:
            # 1 - cos(n_i, n_j) in place of 1 - cos(n_i, -n_j): 2 minus the pair's term
            r = torch.stack([r[0], r[1], 2.0 - r[2]])
        return r.to(verts.device).to(verts.dtype)

    def sdf_value(pts, ratio):
        p = net.sdf(pts, ratio)
        if hold.stepped:
            f = rec.tmp_f32.reshape(-1).double()
            hold.sign_total = f.numel()
            hold.pred = p.detach().reshape(-1).double().clone()
            flip = torch.sign(hold.pred) != torch.sign(f)
            hold.sign_flips = int(flip.sum())
            hold.flip_f64 = hold.pred[flip].abs()
        return p

    tf0 = utils.train_fused

    def train_fused(*a, **k):
        if hold.arm:
            hold.arm = False
            return True
        return tf0(*a, **k)

    def ff(pts, ratio, *a, **k):
        assert hold.stepped and "refine_about" in k, "forward_fused outside the |f| tie"
        return (rec.tmp_f32.to(dtype).clone(),)

    monkeypatch.setattr(net, "discretizeSDF", disc)
    monkeypatch.setattr(net, "_mesh_seed", lambda *a, **k: (bi.clone(), ri.clone(), ci.clone(),
                                                             ps.to(dtype).clone(), ffi))
    monkeypatch.setattr(ops, "mesh_reg_topology", lambda faces, nv: (faces, nv))
    monkeypatch.setattr(ops, "mesh_regularizers", regs)
    monkeypatch.setattr(net, "_sdf_value", sdf_value)
    monkeypatch.setattr(utils, "train_fused", train_fused)
    monkeypatch.setattr(net.sdf, "forward_fused", ff)
    drop = (lambda: [p for n in ("translator", "poses", "trans", "latent") for p in groups(net, data)[n]]) \
        if drop_inner else None
    _wrap_inner_step(monkeypatch, net, hold, lr_scale, drop)
    return hold


def forward_glue(monkeypatch, net, rec, replay_extra=False):
    """Wrap forward_rays to check the arguments forward() hands it against a restatement of the reference's glue
    (network.py:509-543) from the recorded mesh seed: the seed pixels inside the gt mask, subsampled to sample_pix_num
    per frame by one uniform draw each when there are more, then the extra template points TmpVs'[uniform < 4096 / V];
    both draws from the default CPU generator seeded 9 (run_forward), which nothing before them in forward() draws
    from.  The engine run records the pixel set and the extra points; replay_extra (the twin) hands forward_rays the
    engine's extra points (the same vertices), so that the translator's ReLU pattern on them is keyed by the same
    points.  -> namespace: extra_diff, max |twin's own extra points - engine's| (fp32 rounding of the SGD step, unless a
    negative control moves the template)."""
    fr0 = net.forward_rays
    out = types.SimpleNamespace(extra_diff=None)

    def fr(datas, bi, ri, ci, ps, ratio, frame_ids, extra_points=None, **k):
        N = frame_ids.numel()
        sb, sr, sc, sp = rec.seed[:4]
        sel = datas["mask"].to(sb.device)[sb, sr, sc] > 0.
        sb, sr, sc, sp = sb[sel], sr[sel], sc[sel], sp[sel]
        g = torch.Generator().manual_seed(9)
        sample_pix = net.conf.get_int('sample_pix_num')
        if sb.shape[0] > sample_pix * N:
            sel = (torch.rand(sb.shape[0], generator=g) < float(sample_pix * N) / float(sb.shape[0])).to(sb.device)
            sb, sr, sc, sp = sb[sel], sr[sel], sc[sel], sp[sel]
        V = net.TmpVs.shape[0]
        extra = net.TmpVs[(torch.rand(V, generator=g) < 4096. / float(V)).to(sb.device)].detach()
        assert torch.equal(bi, sb) and torch.equal(ri, sr) and torch.equal(ci, sc), "forward()'s pixel set"
        assert torch.equal(ps, sp.to(ps.dtype)), "forward()'s start points"
        assert extra_points is not None and torch.equal(extra_points, extra), "forward()'s extra points"
        if replay_extra:
            assert extra_points.shape == rec.extra.shape
            out.extra_diff = float((extra_points - rec.extra.to(extra_points.dtype)).abs().max())
            extra_points = rec.extra.to(extra_points.dtype).clone()
        else:
            rec.pixels = (bi.clone(), ri.clone(), ci.clone())
            rec.extra = extra_points.detach().clone()
        return fr0(datas, bi, ri, ci, ps, ratio, frame_ids, extra_points=extra_points, **k)
    monkeypatch.setattr(net, "forward_rays", fr)
    return out


def set_level(net, conf, engine):
    """Queue the hierarchy level `conf` (train.coarse / loss_coarse) for the next remesh: on the engine net by
    utils.set_hierarchical_config (which also builds its marching-cubes engine), on the twin directly (its
    discretizeSDF is replayed)."""
    H.dropin()
    import utils
    from selfreconcode_b200 import synth
    if engine:
        loader = torch.utils.data.DataLoader(list(range(net.dataset.poses.shape[0])), 2)
        utils.set_hierarchical_config(conf, 'coarse', net, loader, synth.MC_LADDER_65)
    else:
        net.next_conf = conf.get_config('loss_coarse')
        net.next_train_conf = conf.get_config('train.coarse')


def run_forward(net, data, datas, fids, conf, dtype, engine, hold, sample_pix=2048):
    """A fresh template at level `conf`, then forward() -> backward -> propagateTmpPsGrad.  -> TStep(loss, info,
    parameter gradients per group after backward (direct) and of propagateTmpPsGrad alone (implicit), dL/dTmpPs or
    None, the inner SGD step's displacement -lr * dL/dTmpVs in float64); `hold` is the namespace record_template /
    replay_template returned."""
    from selfreconcode_b200 import train_ops
    flag = train_ops.TC_TRAIN_ENABLED
    train_ops.TC_TRAIN_ENABLED = engine
    try:
        ps = [p for g in groups(net, data).values() for p in g]
        for p in ps:
            p.grad = None
        net.TmpVs = net.Tmpfs = net.TmpOptimizer = None
        net.remesh_time = 0.
        set_level(net, conf, engine)
        datas = {k: v.to(dtype) for k, v in datas.items()}
        with torch.random.fork_rng(devices=[torch.device(DEV)]):
            torch.manual_seed(9)
            loss = net.forward(datas, sample_pix, H.RATIO, fids)
        info = dict(net.info)
        info["pc_loss"] = dict(info["pc_loss"])
        loss.backward()
        direct = flat_grads(net, data)
        dtmp = None if net.TmpPs is None or net.TmpPs.grad is None else net.TmpPs.grad.detach().double().clone()
        for p in ps:
            p.grad = None
        net.propagateTmpPsGrad(fids, H.RATIO)
        info["invInfo"] = net.info["invInfo"]
        return TStep(loss.item(), info, direct, flat_grads(net, data), dtmp, -hold.lr * hold.tmp_grad)
    finally:
        train_ops.TC_TRAIN_ENABLED = flag
