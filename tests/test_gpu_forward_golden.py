"""GPU: one whole optimisation step of the drop-in OptimNetwork -- forward(), loss.backward(), propagateTmpPsGrad()
(train.py:167-169) -- against tests/golden/train_step.npz, which the UNMODIFIED reference produced by running the
same three calls on CPU (oracle/make_golden_r2.py train_step; stand-ins there and here only for what is outside the
path: the point-cloud silhouette renderer and the sample-point generator; the mesh rasteriser is this repo's device
kernel, checked against the fixture's fragments).  Loss terms, converged ray set, dL/dTmpPs, the template vertices
after the inner SGD step and every parameter-gradient digest are compared."""
import types

import numpy as np
import pytest
import torch

from helpers import RATIO, build_render, build_sdf_full, build_skinner, build_translator, dropin, golden, norm_err

pytestmark = pytest.mark.gpu


def fixed_sample_points(pc_input, global_sigma, local_sigma, ratio=6):
    n, d = pc_input.shape
    g = torch.Generator().manual_seed(1000 + n)
    local = pc_input + (torch.randn(n, d, generator=g) * local_sigma).to(pc_input.device)
    if ratio > 0:
        glob = (torch.rand(n // ratio, d, generator=g) * (global_sigma * 2) - global_sigma).to(pc_input.device)
        return torch.cat([local, glob], dim=0)
    return local


class FakePointRenderer:
    """The golden's stand-in for the pytorch3d point silhouette: one soft value per frame."""
    takes_tensors = True
    radius = 0.0

    def __init__(self, H, W):
        self.H, self.W = H, W
        self.rasterizer = types.SimpleNamespace(cameras=None)

    def __call__(self, pts):
        m = torch.sigmoid(2.0 * pts[..., 2].mean(dim=1) + pts[..., 0].mean(dim=1))
        return m.view(-1, 1, 1, 1).expand(-1, self.H, self.W, 1)


def grad_digest(grad, idx):
    flat = grad.detach().double().reshape(-1).cpu()
    r = torch.randn(flat.numel(), generator=torch.Generator().manual_seed(9000 + idx), dtype=torch.float64)
    stride = max(1, flat.numel() // 128)
    return np.concatenate([[flat.norm().item(), (flat * r).sum().item()], flat[::stride][:128].numpy()])


def _build(dev, g):
    dropin()
    from selfreconcode_b200 import synth
    from model.Deformer import CompositeDeformer
    from model.optim import OptimNetwork
    from model.CameraMine import RectifiedPerspectiveCameras
    from model.raster import MeshRasterizer, RasterSettings, SilhouetteRenderer
    import utils
    gd, gs, gr = golden("deform.npz"), golden("sdf_full.npz"), golden("render.npz")
    sdf = build_sdf_full(gs).to(dev)
    comp = CompositeDeformer([build_translator(gd), build_skinner(gd)]).to(dev)
    rn = build_render(gr).to(dev)
    N, H, W = 3, int(g["H"]), int(g["W"])
    cond = [torch.from_numpy(gd[k]).to(dev).requires_grad_(True) for k in ("poses", "trans", "dcond")]
    cam_t = [torch.from_numpy(g[k]).to(dev) for k in ("focals", "pps", "Rs", "Ts")]

    class Data:
        poses, trans = cond[0], cond[1]

        def get_grad_parameters(self, fids, device):
            return cond[0][fids], cond[1][fids], cond[2][fids], None

        def get_camera_parameters(self, n, device):
            return cam_t[0], cam_t[1], cam_t[2], cam_t[3], H, W

        def get_batchframe_data(self, name, fids, batchsize):
            data = getattr(self, name)
            starts = (fids - batchsize // 2).clamp(min=0, max=N - batchsize)
            return data[starts.view(-1, 1) + torch.arange(0, batchsize, device=fids.device).view(1, batchsize)], fids - starts

    cams = RectifiedPerspectiveCameras(*cam_t, image_size=[(W, H)])
    renderer = SilhouetteRenderer(MeshRasterizer(cams, RasterSettings((H, W))))
    conf = synth.Conf(sample_pix_num=100000, grad_weight=0.1, offset_weight=0.05, def_regu=dict(weight=2.0, c=0.5),
                      dct_weight=0.01, color_weight=0.5, normal_weight=0.1, weighted_normal=True)
    net = OptimNetwork(sdf, comp, None, renderer, rn, conf=conf)
    assert abs(net.angThred - float(g["angthr"])) < 1e-6
    net.dataset = Data()
    net.pcRender = FakePointRenderer(H, W)
    net.dctnull = utils.DCTNullSpace(1, 2).to(dev)
    net.TmpVs = torch.from_numpy(g["TmpVs0"]).to(dev).requires_grad_(True)
    net.Tmpfs = torch.from_numpy(g["Tmpfs"]).to(dev)
    net.TmpOptimizer = torch.optim.SGD([net.TmpVs], lr=0.05, momentum=0.9)
    net.forward_time, net.remesh_intersect = 1, 30
    return net, sdf, comp, rn, cond, cams


def test_device_rasteriser_vs_fixture_and_oracle(cuda_dev):
    """csrc/raster.cu on the fixture's deformed template: pix_to_face / barycentrics vs the fragments the oracle
    rasteriser produced for the reference run (same deformed vertices up to fp32 noise of the deformer)."""
    g = golden("train_step.npz")
    net, sdf, comp, rn, cond, cams = _build(cuda_dev, g)
    with torch.no_grad():
        dv = net.deformer(net.TmpVs.detach()[None].expand(3, -1, 3), [cond[2], [cond[0], cond[1]]], ratio=RATIO)
        _, frags = net.maskRender(dv, net.Tmpfs)
    p2f, bary = frags.pix_to_face.cpu().numpy(), frags.bary_coords.cpu().numpy()
    same = p2f == g["pix_to_face"]
    cov = g["pix_to_face"] >= 0
    print("raster: %d covered pixels, %d differ" % (cov.sum(), (~same).sum()))
    assert (~same).sum() <= 0.01 * cov.sum()          # edge pixels can flip with the last bit of a vertex
    assert np.abs(bary - g["bary"])[same & cov].max() < 2e-4
    # the oracle on the SAME screen vertices does the kernel's fp32 arithmetic in the same order: bit-exact face ids,
    # barycentrics and depth
    from oracle import oracle as O
    vs = net.maskRender.rasterizer.screen_vertices(dv)
    zbuf = frags.zbuf.cpu().numpy()
    for n in range(3):
        po, bo, zo = O.raster_mesh(vs[n].cpu().numpy(), net.Tmpfs.cpu().numpy(), int(g["H"]), int(g["W"]))
        pg = p2f[n, :, :, 0]
        pg = np.where(pg >= 0, pg - n * net.Tmpfs.shape[0], pg)
        assert np.array_equal(pg, po), (n, (pg != po).sum())
        assert np.array_equal(bary[n, :, :, 0].view(np.uint32), bo.view(np.uint32)), n
        assert np.array_equal(zbuf[n, :, :, 0].view(np.uint32), zo.view(np.uint32)), n


def _run_step(cuda_dev, g, fused):
    from selfreconcode_b200 import train_ops
    net, sdf, comp, rn, cond, cams = _build(cuda_dev, g)
    import utils
    import model.optim as mo
    saved = utils.sample_points, mo.utils.sample_points
    frags = types.SimpleNamespace(pix_to_face=torch.from_numpy(g["pix_to_face"]).to(cuda_dev),
                                  bary_coords=torch.from_numpy(g["bary"]).to(cuda_dev))
    net.raster_seed = lambda dv, tv, tf, cam: frags          # the reference run's own fragments: same seeds
    datas = {"img": torch.from_numpy(g["img"]).to(cuda_dev), "mask": torch.ones(3, int(g["H"]), int(g["W"]), device=cuda_dev),
             "normal": torch.from_numpy(g["normal"]).to(cuda_dev)}
    fids = torch.arange(3, device=cuda_dev)
    torch.manual_seed(123)
    utils.sample_points = fixed_sample_points
    mo.utils.sample_points = fixed_sample_points
    train_ops.TC_TRAIN_ENABLED = fused
    try:
        loss = net.forward(datas, 100000, RATIO, fids)
        info = dict(net.info)
        loss.backward()
        tmpps, gl = net.TmpPs.detach().clone(), net.TmpPs.grad.detach().clone()
        net.propagateTmpPsGrad(fids, RATIO)
    finally:
        train_ops.TC_TRAIN_ENABLED = True
        utils.sample_points, mo.utils.sample_points = saved    # later tests draw from the real sampler's stream
    named = [("sdf." + k, q) for k, q in sorted(sdf.named_parameters())] + \
            [("def." + k, q) for k, q in sorted(comp.named_parameters())] + \
            [("rn." + k, q) for k, q in sorted(rn.named_parameters())] + list(zip(("poses", "trans", "dcond"), cond))
    worst = {}
    for i, (k, q) in enumerate(named):
        if ("g__" + k) not in g.files:
            assert q.grad is None or float(q.grad.abs().max()) == 0, k
            continue
        assert q.grad is not None, k
        d, r = grad_digest(q.grad, i), g["g__" + k]
        # (relative difference of the norms and of the 128 strided samples, reference norm of the tensor)
        worst[k] = (max(abs(d[0] - r[0]) / max(r[0], 1e-12), np.abs(d[2:] - r[2:]).max() / max(np.abs(r[2:]).max(), 1e-12)),
                    float(r[0]))
    return net, loss, info, tmpps, gl, worst


def test_optimisation_step_vs_reference_golden(cuda_dev):
    g = golden("train_step.npz")
    # the torch-autograd twin first (fp32 cuBLAS, create_graph double backward): how far two fp32 evaluations of this
    # step are from one another is the yardstick for the tensor-core engine's numbers below
    _, loss_t, info_t, _, gl_t, worst_t = _run_step(cuda_dev, g, False)
    net, loss, info, tmpps, gl, worst = _run_step(cuda_dev, g, True)
    # ---- ray set
    key = lambda b, r, c: set(zip(b.tolist(), r.tolist(), c.tolist()))
    mine = key(net.batch_inds.cpu().numpy(), net.row_inds.cpu().numpy(), net.col_inds.cpu().numpy())
    ref = key(g["batch_inds"], g["row_inds"], g["col_inds"])
    print("rays: traced %s (reference %s); converged set: %d common, %d only here, %d only reference"
          % (info["rayInfo"], tuple(g["rayinfo"]), len(mine & ref), len(mine - ref), len(ref - mine)))
    assert info["rayInfo"][0] == int(g["rayinfo"][0])
    diff = len(mine ^ ref)
    assert diff <= 4
    same_set = diff == 0
    tol = 1.0 if same_set else 25.0          # a ray more or less moves every per-frame mean by ~1/170
    # ---- losses
    terms = {k: (info[k], float(g["info_" + k])) for k in ("grad_loss", "offset_loss", "def_loss", "dct_loss",
                                                          "color_loss", "normal_loss", "pc_loss_sdf")}
    terms["mask_loss"] = (info["pc_loss"]["mask_loss"], float(g["info_mask_loss"]))
    terms["total"] = (loss.item(), float(g["loss"]))
    print({k: "%.6f / %.6f" % v for k, v in terms.items()}, "twin total %.6f" % loss_t.item())
    # pc_loss_sdf = mean |f| over the template vertices (~1e-3): the tensor-core engine's ~1e-6 absolute error on f
    # shows there, and 60x (the term's weight) in the total
    atol = {"pc_loss_sdf": 5e-6, "total": 60 * 5e-6}
    for k, (a, b) in terms.items():
        assert abs(a - b) < tol * 3e-4 * max(abs(b), 1e-3) + atol.get(k, 0.0), (k, a, b)
    np.testing.assert_allclose(net.TmpVs.detach().cpu().numpy(), g["TmpVs_after"], atol=2e-6)
    if same_set:
        order = np.lexsort((net.col_inds.cpu().numpy(), net.row_inds.cpu().numpy(), net.batch_inds.cpu().numpy()))
        order_r = np.lexsort((g["col_inds"], g["row_inds"], g["batch_inds"]))
        assert np.abs(tmpps.cpu().numpy()[order] - g["tmpps"][order_r]).max() < 7e-5
        e = norm_err(gl.cpu().numpy()[order], g["grad_l_p"][order_r])
        et = norm_err(gl_t.cpu().numpy()[order], g["grad_l_p"][order_r])
        print("dL/dTmpPs norm-wise err: tensor-core engine %.2e, torch twin %.2e" % (e, et))
        assert e < 5e-3
        assert tuple(net.info["invInfo"]) == tuple(g["invinfo"])
    # ---- parameter gradients (digests: norm, random projection, 128 strided samples)
    # per module: every tensor's relative difference weighted by its share of the module's gradient norm (a tensor whose
    # exact gradient vanishes -- e.g. the scale of f under the normalised-normal loss -- carries no weight)
    def module_err(w, grp):
        num = sum((w[k][0] * w[k][1]) ** 2 for k in w if k.split(".")[0] == grp)
        den = sum(w[k][1] ** 2 for k in w if k.split(".")[0] == grp)
        return float(np.sqrt(num / max(den, 1e-300)))

    groups = {grp: (module_err(worst, grp), module_err(worst_t, grp)) for grp in ("sdf", "def", "rn", "poses", "trans", "dcond")}
    print("parameter gradients vs the reference, norm-weighted relative difference per module "
          "[tensor-core engine, torch twin]:", {k: ["%.1e" % v for v in vs] for k, vs in groups.items()})
    top = sorted(worst.items(), key=lambda kv: -kv[1][0] * kv[1][1])[:10]
    print("largest contributions (tensor, rel diff, reference norm, twin rel diff):")
    for k, (e, n) in top:
        print("   %-28s %.1e  %.2e  twin %.1e" % (k, e, n, worst_t[k][0]))
    # ReLU networks (rendering network, translator): two correct evaluations differ on the units whose pre-activation
    # is within rounding of 0, which moves a 174-ray gradient by per cent -- the twin shows the same against the reference
    for grp in ("def", "poses", "trans", "dcond"):
        assert groups[grp][0] < tol * 2e-2, (grp, groups[grp])
    assert groups["rn"][0] < max(3 * groups["rn"][1], tol * 2e-2), groups["rn"]
    assert groups["sdf"][0] < max(3 * groups["sdf"][1], tol * 2e-2), groups["sdf"]
