"""CPU: the autograd wiring of the twice-differentiable sampler and of the upsample op
(dropin/MCAcc/_autograd.py), with torch's own CPU ops substituted for the CUDA extension modules:
first- and second-order gradcheck in float64 -- the reference's own check for these wrappers
(MCAcc/check_grid_sampler_mine.py:11,16)."""
import sys
import types

import pytest
import torch
import torch.nn.functional as F

import helpers as H


def _manual_sample(inp, grid):
    """trilinear, border padding, align_corners=False from elementary differentiable ops (torch's own
    grid_sampler_3d has no double backward -- the reason the reference ships its sampler)."""
    N, C, D, Hh, W = inp.shape
    out_shape = grid.shape[1:4]
    g = grid.reshape(N, -1, 3)
    size = torch.tensor([W, Hh, D], dtype=inp.dtype)
    pos = ((g + 1) * size - 1) / 2
    pos = torch.minimum(torch.maximum(pos, torch.zeros_like(pos)), (size - 1).expand_as(pos))
    lo = pos.detach().floor()
    fr = pos - lo
    lo = lo.long()
    hi = torch.minimum(lo + 1, (size - 1).long().expand_as(lo))
    res = 0
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                ix = (hi if dx else lo)[..., 0]
                iy = (hi if dy else lo)[..., 1]
                iz = (hi if dz else lo)[..., 2]
                wgt = (fr[..., 0] if dx else 1 - fr[..., 0]) * (fr[..., 1] if dy else 1 - fr[..., 1]) * \
                      (fr[..., 2] if dz else 1 - fr[..., 2])
                vals = torch.stack([inp[n][:, iz[n], iy[n], ix[n]] for n in range(N)], 0)   # [N,C,P]
                res = res + vals * wgt.unsqueeze(1)
    return res.reshape(N, C, *out_shape)


def _fake_sampler():
    m = types.ModuleType("GridSamplerMine")

    def fwd(inp, grid, interp=0, pad=1):
        return _manual_sample(inp, grid)

    def bwd(inp, grid, gout, interp=0, pad=1):
        with torch.enable_grad():
            i, g = inp.detach().requires_grad_(True), grid.detach().requires_grad_(True)
            gi, gg = torch.autograd.grad(fwd(i, g), (i, g), gout)
        return gi, gg

    def dbwd(ggi, ggg, inp, grid, gout, interp=0, pad=1):
        with torch.enable_grad():
            i, g, o = (t.detach().requires_grad_(True) for t in (inp, grid, gout))
            gi, gg = torch.autograd.grad(fwd(i, g), (i, g), o, create_graph=True)
            s = (gi * ggi).sum() + (gg * ggg).sum()
            di, dg, do = torch.autograd.grad(s, (i, g, o), allow_unused=True)
        z = lambda t, like: torch.zeros_like(like) if t is None else t
        return z(di, inp), z(dg, grid), z(do, gout)

    m.forward, m.backward, m.dbackward = fwd, bwd, dbwd
    return m


def test_sampler_wrapper_first_and_second_order(monkeypatch):
    H.dropin()
    monkeypatch.setitem(sys.modules, "GridSamplerMine", _fake_sampler())
    from MCAcc import GridSamplerMine3dFunction
    g = torch.Generator().manual_seed(0)
    vol = torch.randn(1, 3, 4, 5, 6, dtype=torch.float64, generator=g, requires_grad=True)
    # keep sample points away from cell faces (the sampler is only piecewise smooth)
    base = torch.rand(1, 1, 1, 7, 3, dtype=torch.float64, generator=g) * 1.2 - 0.6
    grid = base.clone().requires_grad_(True)
    fn = lambda v, q: GridSamplerMine3dFunction.apply(v, q)
    assert torch.allclose(fn(vol, grid), F.grid_sample(vol, grid, mode="bilinear", padding_mode="border",
                                                       align_corners=False))
    assert torch.autograd.gradcheck(fn, (vol, grid), eps=1e-6, atol=1e-6)
    assert torch.autograd.gradgradcheck(fn, (vol, grid), eps=1e-6, atol=1e-5)
    with pytest.raises(NotImplementedError):
        GridSamplerMine3dFunction.apply(vol, grid, 'bilinear', 'border', True)


def test_upsample_wrapper_gradient(monkeypatch):
    H.dropin()
    m = types.ModuleType("interp2x_boundary3d")

    def fwd(x, balance):
        b, c, d, h, w = x.shape
        up = F.interpolate(x, size=(2 * d - 1, 2 * h - 1, 2 * w - 1), mode="trilinear", align_corners=True)
        return [up, up > balance]

    def bwd(g):
        b, c, od, oh, ow = g.shape
        with torch.enable_grad():
            x = torch.zeros(b, c, (od + 1) // 2, (oh + 1) // 2, (ow + 1) // 2, dtype=g.dtype, requires_grad=True)
            (gx,) = torch.autograd.grad(fwd(x, 0.0)[0], x, g)
        return gx

    m.forward, m.backward = fwd, bwd
    monkeypatch.setitem(sys.modules, "interp2x_boundary3d", m)
    from MCAcc.interp2x_boundary3d import Interp2xBoundary3d, Interp2xBoundary3dFunction
    x = torch.randn(1, 1, 3, 4, 3, dtype=torch.float64, requires_grad=True)
    out, flag = Interp2xBoundary3d(0.1)(x)
    assert out.shape == (1, 1, 5, 7, 5) and flag.dtype == torch.bool and not flag.requires_grad
    assert torch.autograd.gradcheck(lambda t: Interp2xBoundary3dFunction.apply(t, 0.1)[0], (x,), eps=1e-6, atol=1e-6)


def test_index_rows_first_and_second_order():
    """model/_fused.index_rows (the per-point gather of per-frame poses, translations and latent codes) and
    scatter_rows (the per-frame mean of the ray losses): the values of index_select / a per-frame sum, and first- and
    second-order gradcheck in float64."""
    H.dropin()
    from model._fused import index_rows, scatter_rows
    g = torch.Generator().manual_seed(0)
    t = torch.randn(3, 4, 5, dtype=torch.float64, generator=g).requires_grad_(True)
    idx = torch.tensor([2, 0, 2, 2, 1, 0, 2])
    assert torch.equal(index_rows(t, idx), t.index_select(0, idx))
    assert torch.autograd.gradcheck(lambda t: index_rows(t, idx), (t,))
    assert torch.autograd.gradgradcheck(lambda t: index_rows(t, idx) ** 2, (t,))
    s = torch.randn(7, 2, dtype=torch.float64, generator=g).requires_grad_(True)
    ref = torch.stack([s[idx == i].sum(0) for i in range(4)])
    assert torch.allclose(scatter_rows(s, idx, 4), ref, rtol=0, atol=1e-15)
    assert torch.autograd.gradcheck(lambda s: scatter_rows(s, idx, 4) ** 2, (s,))
