"""One optimisation step through the OptimNetwork drop-in on synthetic data (train.py:150-171's
sequence: forward -> backward -> propagateTmpPsGrad -> optimizer.step), plus the ray part of
infer() and discretizeSDF.  Component parity lives in test_gpu_parity / test_optim_propagate; here
the sequence is checked for self-consistency on the GPU."""
import types

import numpy as np
import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu


def build(n_frames=2, Hh=96, Ww=96):
    H.dropin()
    from selfreconcode_b200 import synth
    from model.Deformer import CompositeDeformer
    from model.optim import OptimNetwork
    from model.CameraMine import RectifiedPerspectiveCameras
    from MCAcc import Seg3dLossless
    dev = "cuda"
    sdf = synth.make_sdf().to(dev)
    comp = CompositeDeformer([synth.make_translator(), synth.make_skinner(resolution=(33, 57, 17))]).to(dev)
    rn = synth.make_render().to(dev)
    data = synth.SyntheticDataset(n_frames, Hh, Ww).to(dev)
    cam = synth.camera(Hh, Ww)
    fids = torch.arange(n_frames, device=dev)
    poses, trans, dcond, _ = data.get_grad_parameters(fids, dev)
    with torch.no_grad():
        rays = synth.make_rays(cam, n_frames,
                               lambda p: sdf.forward_fused(p.to(dev), H.RATIO, False, False)[0].view(-1),
                               lambda p, b: comp.forward_fused(p.to(dev), [dcond, [poses, trans]], b.to(dev), H.RATIO)[0])
    f, pp, R, T, _, _ = data.get_camera_parameters(n_frames, dev)
    cams = RectifiedPerspectiveCameras(f.detach(), pp.detach(), R, T.detach(), image_size=[(Ww, Hh)])
    holder = types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=cams))
    eng = Seg3dLossless(query_func=None, b_min=[-0.9, -0.9, -0.9], b_max=[0.9, 0.9, 0.9],
                        resolutions=[(9, 9, 9), (17, 17, 17), (33, 33, 33), (65, 65, 65)],
                        align_corners=False, balance_value=0.0, use_cuda_impl=True).to(dev)
    conf = synth.Conf(grad_weight=0.1, color_weight=0.5, normal_weight=0.0)
    net = OptimNetwork(sdf, comp, eng, holder, rn, conf=conf)
    net.dataset = data
    # the raster seed of the real pipeline puts D(start) on the pixel's own ray; here the seed is a
    # Gauss-Newton solve of {f(p) = 0, (D(p) - c) x v = 0} along the pixel rays (test-side torch
    # on top of the fused value / gradient / Jacobian kernels), keeping the pixels where it settles
    import utils
    bi, ri, ci = rays["batch_inds"].to(dev), rays["rows"].to(dev), rays["cols"].to(dev)
    pix = torch.stack([ci, ri, torch.ones_like(ci)], dim=1).float()
    dc = [dcond.detach(), [poses.detach(), trans.detach()]]
    with torch.no_grad():
        v = cams.to(dev).view_rays(pix)
        c = cams.cam_pos().view(1, 3)
        p = rays["pstar"].to(dev).clone()
        vx = torch.zeros(p.shape[0], 3, 3, device=dev)
        vx[:, 0, 1], vx[:, 0, 2], vx[:, 1, 0] = -v[:, 2], v[:, 1], v[:, 2]
        vx[:, 1, 2], vx[:, 2, 0], vx[:, 2, 1] = -v[:, 0], -v[:, 1], v[:, 0]
        for _ in range(12):
            f, gf, _ = sdf.forward_fused(p, H.RATIO, want_grad=True, want_feat=False)
            d, J, _ = comp.forward_fused(p, dc, bi, H.RATIO, want_jac=True)
            res = torch.cat([f.view(-1, 1), torch.cross(v, d - c, dim=1)], dim=1)        # [P,4]
            B = torch.cat([gf.view(-1, 1, 3), vx @ J], dim=1)                           # [P,4,3]
            step = torch.linalg.solve(B.transpose(1, 2) @ B + 1e-9 * torch.eye(3, device=dev),
                                      (B.transpose(1, 2) @ res.unsqueeze(-1)))
            p = p - step.squeeze(-1).clamp(-0.05, 0.05)
        seed, ok = utils.OptimizeSurfacePs(cams.cam_pos(), v, p.clone(), bi, sdf, H.RATIO, comp, dc, dthreshold=2e-5,
                                           athreshold=0.5 * net.angThred, w1=3.05, w2=1., times=5)
    assert int(ok.sum()) > 0.8 * ok.numel(), (int(ok.sum()), ok.numel())
    g = torch.Generator().manual_seed(3)
    jit = 2e-4 * torch.randn(int(ok.sum()), 3, generator=g).to(dev)
    rays = dict(batch_inds=bi[ok], rows=ri[ok], cols=ci[ok], pstar=seed[ok], init_pts=seed[ok] + jit)
    return net, data, rays, fids


def test_training_step_sequence():
    net, data, rays, fids = build()
    dev = "cuda"
    N, Hh, Ww = fids.numel(), data.H, data.W
    params = list(net.sdf.parameters()) + list(net.deformer.parameters()) + list(net.netRender.parameters()) \
        + list(data.parameters())
    opt = torch.optim.Adam([q for q in params if q.requires_grad], lr=1e-4)
    before = [q.detach().clone() for q in net.sdf.parameters()]
    img = torch.rand(N, Hh, Ww, 3, device=dev) * 2 - 1
    # the traced pixel set: aim rays from the pixel grid so that view_rays(pix) is the ray
    bi, ri, ci = rays["batch_inds"].to(dev), rays["rows"].to(dev), rays["cols"].to(dev)
    loss = net.forward_rays({"img": img}, bi, ri, ci, rays["init_pts"].to(dev).clone(), H.RATIO, fids)
    assert torch.isfinite(loss)
    total, conv = net.info["rayInfo"]
    assert total == bi.numel() and conv > 0.1 * total, net.info
    opt.zero_grad()
    loss.backward()
    assert net.TmpPs.grad is not None and float(net.TmpPs.grad.abs().max()) > 0
    g_before = net.sdf.lin3.weight_v.grad.detach().clone()
    net.propagateTmpPsGrad(fids, H.RATIO)
    tot, ok = net.info["invInfo"]
    assert tot == conv and ok > 0.9 * tot
    # the implicit-differentiation term reaches the sdf, the translator and the per-frame codes
    assert float((net.sdf.lin3.weight_v.grad - g_before).abs().max()) > 0
    assert float(net.deformer.defs[0].lin0.weight.grad.abs().max()) > 0
    assert float(data.poses.grad.abs().max()) > 0 and float(data.conds[0].grad.abs().max()) > 0
    for q in params:
        if q.grad is not None:
            assert torch.isfinite(q.grad).all()
    opt.step()
    assert any(float((a - b).abs().max()) > 0 for a, b in zip(before, net.sdf.parameters()))
    # folded weights must follow the optimiser step (FoldCache keyed on Tensor._version)
    p = rays["pstar"][:64].to(dev)
    with torch.no_grad():
        fused = net.sdf.forward_fused(p, H.RATIO, False, False)[0].view(-1)
    plain = net.sdf(p.clone().requires_grad_(True), H.RATIO).view(-1)
    assert H.rel_err(fused.cpu().numpy(), plain.detach().cpu().numpy()) < 1e-4


def test_infer_rays_and_discretize():
    net, data, rays, fids = build()
    dev = "cuda"
    bi, ri, ci = rays["batch_inds"].to(dev), rays["rows"].to(dev), rays["cols"].to(dev)
    colors = net.infer_rays(bi, ri, ci, rays["init_pts"].to(dev), data.H, data.W, H.RATIO, fids)
    assert colors.shape == (fids.numel(), data.H, data.W, 3)
    assert float(colors.min()) >= 0 and float(colors.max()) <= 255
    bg = torch.ones_like(colors[..., 0], dtype=torch.bool)
    bg[bi, ri, ci] = False
    assert float((colors[bg] - 255.).abs().max()) == 0
    assert float((colors[~bg] - 255.).abs().max()) > 0
    verts, faces = net.discretizeSDF(H.RATIO, None, 0.0)
    assert verts.shape[0] > 100 and faces.shape[0] > 100 and int(faces.max()) == verts.shape[0] - 1
    with torch.no_grad():
        f = net.sdf.forward_fused(verts, H.RATIO, False, False)[0].view(-1)
    assert float(f.abs().max()) < 5e-3   # vertices sit on the zero set up to the linear edge interpolation (65^3 grid)


def _one_step(net, data, rays, fids, fused, conf):
    """forward_rays (eikonal + colour + normal + def_regu + offset) -> backward -> propagateTmpPsGrad with the
    training evaluations on the tensor-core training engine (fused) or on torch autograd (cuBLAS)."""
    from selfreconcode_b200 import train_ops
    dev = "cuda"
    N, Hh, Ww = fids.numel(), data.H, data.W
    train_ops.TC_TRAIN_ENABLED = fused
    net.conf = conf
    g = torch.Generator().manual_seed(5)
    img = (torch.rand(N, Hh, Ww, 3, generator=g) * 2 - 1).to(dev)
    nrm = torch.nn.functional.normalize(torch.randn(N, Hh, Ww, 3, generator=g), dim=-1).to(dev)
    params = [q for q in list(net.sdf.parameters()) + list(net.deformer.parameters()) +
              list(net.netRender.parameters()) + list(data.parameters()) if q.requires_grad]
    for q in params:
        q.grad = None
    torch.manual_seed(9)     # sample_points draws from the global generators
    bi, ri, ci = rays["batch_inds"].to(dev), rays["rows"].to(dev), rays["cols"].to(dev)
    loss = net.forward_rays({"img": img, "normal": nrm}, bi, ri, ci, rays["init_pts"].to(dev).clone(), H.RATIO, fids)
    info = dict(net.info)
    loss.backward()
    gp = net.TmpPs.grad.detach().clone()
    net.propagateTmpPsGrad(fids, H.RATIO)
    grads = [q.grad.detach().clone() if q.grad is not None else None for q in params]
    return loss.item(), info, gp, grads, params


def test_training_step_fused_vs_autograd():
    """The same optimisation step twice on the same GPU: training evaluations through the tensor-core training
    engine (forward tangents + one reverse sweep, wgmma weight-gradient GEMMs) vs the torch-autograd twin
    (create_graph=True double backward on cuBLAS): loss terms, dL/dTmpPs and every parameter gradient agree."""
    from selfreconcode_b200 import synth, train_ops
    net, data, rays, fids = build()
    conf = synth.Conf(grad_weight=0.1, color_weight=0.5, normal_weight=0.1, weighted_normal=True, offset_weight=0.05,
                      def_regu=dict(weight=2.0, c=0.5))
    try:
        la, ia, ga, gra, params = _one_step(net, data, rays, fids, False, conf)
        lf, inf, gf, grf, _ = _one_step(net, data, rays, fids, True, conf)
    finally:
        train_ops.TC_TRAIN_ENABLED = True
    print("loss autograd %.6f fused %.6f" % (la, lf), {k: (ia[k], inf[k]) for k in ia if k.endswith("_loss")})
    assert abs(la - lf) < 2e-4 * max(1.0, abs(la))
    for k in ("grad_loss", "color_loss", "normal_loss", "def_loss", "offset_loss"):
        assert abs(ia[k] - inf[k]) < 2e-4 * max(1.0, abs(ia[k])), (k, ia[k], inf[k])
    assert H.norm_err(gf.cpu().numpy(), ga.cpu().numpy()) < 2e-3
    names = [n for n, q in list(net.sdf.named_parameters()) + list(net.deformer.named_parameters()) +
             list(net.netRender.named_parameters()) + list(data.named_parameters()) if q.requires_grad]
    worst = {}
    for n, a, f in zip(names, gra, grf):
        assert (a is None) == (f is None), n
        if a is not None and float(a.abs().max()) > 0:
            worst[n] = H.norm_err(f.cpu().numpy(), a.cpu().numpy())
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:6]
    print("largest gradient differences:", top)
    sdf_names = {n for n, _ in net.sdf.named_parameters()}
    first_order = {k: v for k, v in worst.items() if k not in sdf_names or k.startswith(("defs.", "poses", "trans", "conds"))}
    # SDF parameters: second-order terms through softplus(beta=100) (DESIGN.md section 4); everything else first order
    assert max(worst.values()) < 5e-2, top
