"""GPU: the IGR pre-fit of the template SDF (OptimNetwork.initializeTmpSDF) on the tensor-core training engine against
the reference's autograd loop, which SELFRECON_B200_TC_TRAIN=0 and non-stock modules keep.

Template: the marching-cubes vertices of synth.make_sdf()'s zero set, with and without vertex normals.
  * one step on fixed points vs a float64 copy of the module through the autograd loop: each loss term within 1e-4
    relative, and the SDF parameter gradients within 1e-4 as ||g - g64|| / ||g64|| over the module (the fp32 autograd
    loop's figure is printed beside it);
  * 100-epoch fits from seeds 0-2 on both paths: the mean over the seeds of the engine's mean |f| on the vertices and
    of its eikonal residual each within 1.5x of the fp32 loop's largest (see test_fit_100_epochs)."""
import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu
DEV = "cuda"

_TEMPLATE = {}


def template():
    """(a fresh synth.make_sdf() module, vertices [V,3], unit vertex normals [V,3]): the template is the 97^3
    marching-cubes mesh of the module's zero set over [-1.2, 1.2]^3."""
    if not _TEMPLATE:
        H.dropin()
        from selfreconcode_b200 import ops, synth
        sdf = synth.make_sdf().to(DEV)
        n, lo, step = 97, -1.2, 2.4 / 96
        ax = torch.arange(n, device=DEV, dtype=torch.float32) * step + lo
        zz, yy, xx = torch.meshgrid(ax, ax, ax, indexing="ij")
        pts = torch.stack([xx, yy, zz], -1).reshape(-1, 3)
        with torch.no_grad():
            grid = torch.cat([sdf.forward_fused(p, 1.0, False, False)[0] for p in torch.split(pts, 1 << 18)])
        v, f = ops.marching_cubes(grid.reshape(n, n, n).contiguous(), step, step, step, lo, lo, lo, 0.0)
        v, f = v.float().contiguous(), f.long()
        fn = torch.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]], dim=1)
        vn = torch.zeros_like(v).index_add(0, f.reshape(-1), fn.repeat_interleave(3, 0))
        vn = vn / vn.norm(dim=1, keepdim=True).clamp(min=1e-12)
        _TEMPLATE.update(v=v, n=vn)
        print("template: %d vertices" % v.shape[0])
    from selfreconcode_b200 import synth
    return synth.make_sdf().to(DEV), _TEMPLATE["v"], _TEMPLATE["n"]


def optnet(sdf, v, n):
    from model.optim import OptimNetwork
    on = OptimNetwork(sdf, None, None, None, None)
    on.tmpBodyVs, on.tmpBodyNs = v, n
    return on


def _grads(module):
    return [p.grad.detach().double().reshape(-1) if p.grad is not None else torch.zeros(p.numel(), device=DEV,
                                                                                         dtype=torch.float64)
            for p in module.parameters()]


def _step(sdf, on_pts, off_pts, normals, with_normals, engine, monkeypatch):
    from selfreconcode_b200 import train_ops
    monkeypatch.setattr(train_ops, "TC_TRAIN_ENABLED", engine)
    net = optnet(sdf, on_pts, normals)
    sdf.zero_grad()
    loss, m, g, nl = net.igr_losses(on_pts, off_pts, normals, with_normals)
    loss.backward()
    return [float(t) for t in (loss, m, g, nl.sum())], _grads(sdf)


@pytest.mark.parametrize("with_normals", [False, True])
def test_one_step_vs_float64(with_normals, monkeypatch):
    H.dropin()
    import utils
    sdf, v, n = template()
    torch.manual_seed(0)
    perm = torch.randperm(v.shape[0])[:5000].to(DEV)
    on, nrm = v[perm].contiguous(), n[perm].contiguous()
    off = utils.sample_points(on, 1.8, 0.01)
    eng, g_eng = _step(sdf, on, off, nrm, with_normals, True, monkeypatch)
    a32, g_a32 = _step(sdf, on, off, nrm, with_normals, False, monkeypatch)
    from selfreconcode_b200 import synth
    sdf64 = synth.make_sdf().double().to(DEV)
    a64, g_64 = _step(sdf64, on.double(), off.double(), nrm.double(), with_normals, False, monkeypatch)
    terms = ["loss", "manifold", "eikonal", "normals"]
    for name, x, y, z in zip(terms, eng, a32, a64):
        if name == "normals" and not with_normals:
            continue
        print("%-9s engine %.9e  autograd32 %.9e  float64 %.9e  rel %.2e" % (name, x, y, z, abs(x - z) / abs(z)))
        assert abs(x - z) <= 1e-4 * abs(z), name

    def gerr(g):
        num = sum(float(((a - b) ** 2).sum()) for a, b in zip(g, g_64))
        den = sum(float((b ** 2).sum()) for b in g_64)
        return (num / den) ** 0.5

    e_eng, e_a32 = gerr(g_eng), gerr(g_a32)
    print("parameter gradients vs float64: engine %.2e, fp32 autograd loop %.2e" % (e_eng, e_a32))
    assert e_eng <= 1e-4


def _fit(engine, with_normals, epochs, monkeypatch, seed=0):
    from selfreconcode_b200 import train_ops
    sdf, v, n = template()
    net = optnet(sdf, v, n)
    monkeypatch.setattr(train_ops, "TC_TRAIN_ENABLED", engine)
    torch.manual_seed(seed)
    net.initializeTmpSDF(epochs, None, with_normals)
    return sdf


def _fit_metrics(sdf, v, monkeypatch):
    """(mean |f| on the vertices, mean (|grad f| - 1)^2 on fixed off-surface samples), on the fp32 autograd path."""
    from selfreconcode_b200 import train_ops
    H.dropin()
    import utils
    monkeypatch.setattr(train_ops, "TC_TRAIN_ENABLED", False)
    torch.manual_seed(123)
    off = utils.sample_points(v, 1.8, 0.01).requires_grad_()
    x = v.detach().requires_grad_()
    f = sdf(x, -1)
    g = sdf.gradient(off, sdf(off, -1))
    return float(f.abs().mean()), float(((g.norm(dim=-1) - 1) ** 2).mean())


@pytest.mark.parametrize("with_normals", [False, True])
def test_fit_100_epochs(with_normals, monkeypatch):
    """Seeds 0-2 on both paths.  A single fit is not reproducible run to run (Adam amplifies the last-bit differences
    of atomically accumulated gradients), and on the H100 one seed's eikonal residual moved by 2x between two runs of
    the same path, so the bar sits outside that spread: the engine's mean over the seeds within 1.5x of the autograd
    loop's largest."""
    _, v, _ = template()
    got = {True: [], False: []}
    for seed in (0, 1, 2):
        for engine in (True, False):
            sdf = _fit(engine, with_normals, 100, monkeypatch, seed)
            got[engine].append(_fit_metrics(sdf, v, monkeypatch))
    for i, name in enumerate(("mean|f|", "eikonal")):
        e, a = [m[i] for m in got[True]], [m[i] for m in got[False]]
        print("100 epochs (normals=%s) %s: engine %s; autograd loop %s" %
              (with_normals, name, " ".join("%.3e" % x for x in e), " ".join("%.3e" % x for x in a)))
        assert sum(e) / len(e) <= 1.5 * max(a), name
