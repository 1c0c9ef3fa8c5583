"""CPU: the float64 restatement of the trilinear sampler (tests/grid_sampler_ref.py) against torch's own float64
grid_sample away from ties, gradcheck / gradgradcheck, closed forms, and negative controls -- variants of the x,
floor and mask rule that must fail the device bars (corner indices exact; grad_grid exactly 0 where the mask is 0;
|a - b| <= BAR * mag)."""
import pytest
import torch
import torch.nn.functional as F

import grid_sampler_ref as R


def _inputs(N=2, C=3, D=5, H=6, W=7, P=300, lo=-1.2, hi=1.2, dtype=torch.float64, seed=0):
    g = torch.Generator().manual_seed(seed)
    vol = torch.randn(N, C, D, H, W, generator=g, dtype=torch.float64).to(dtype)
    grid = (lo + (hi - lo) * torch.rand(N, P, 3, generator=g, dtype=torch.float64)).to(dtype)
    go = torch.randn(N, C, P, generator=g, dtype=torch.float64).to(dtype)
    ggi = torch.randn(N, C, D, H, W, generator=g, dtype=torch.float64).to(dtype)
    ggg = torch.randn(N, P, 3, generator=g, dtype=torch.float64).to(dtype)
    return vol, grid, go, ggi, ggg


def _away_from_kinks(grid, sizes, margin=1e-3):
    """Rows of grid [N,P,3] whose x on every axis is `margin` away from an integer and from the border."""
    keep = torch.ones(grid.shape[:2], dtype=torch.bool)
    for k, s in enumerate(sizes):
        x = R.unnormalise(grid[..., k], s).double()
        keep &= ((x - x.round()).abs() > margin) & ((x.abs() > margin) & ((x - (s - 1)).abs() > margin))
    return keep


def _torch_sample(vol, grid):
    return F.grid_sample(vol, grid.unsqueeze(1).unsqueeze(1), mode="bilinear", padding_mode="border",
                         align_corners=False).flatten(2)


def _all_outputs(vol, grid, go, ggi, ggg):
    """{name: (value, mag)} of every restatement output, and the corner indices."""
    out = {"fwd": R.forward(vol, grid)}
    (gi, gg) = R.backward(vol, grid, go)
    out.update(bwd_input=gi, bwd_grid=gg)
    (a, b, c) = R.dbackward(ggi, ggg, vol, grid, go)
    out.update(dbwd_input=a, dbwd_grid=b, dbwd_gout=c)
    return out, R.corner_index(vol, grid)


def _fails(variant, correct, dtype, masks=None):
    """The device bars the variant's outputs fail: 'index', 'zero' and '<name>' (with their ratio)."""
    (vo, vi), (co, ci) = variant, correct
    failed = {}
    if not torch.equal(vi, ci):
        failed["index"] = int((vi != ci).any(-1).sum())
    if masks is not None:
        for name in ("bwd_grid", "dbwd_grid"):
            if bool((vo[name][0][masks == 0] != 0).any()):
                failed["zero"] = True
    for name, (b, mag) in co.items():
        r = R.bar_ratio(vo[name][0], b, mag)
        if not r <= R.BAR[dtype]:
            failed[name] = r
    return failed


def _masks(vol, grid):
    N, _, D, H, W = vol.shape
    return torch.stack([a[2] for a in R.axes(grid.reshape(N, -1, 3), (W, H, D))], dim=-1)


def test_matches_torch_grid_sample_away_from_ties():
    vol, grid, go, _, _ = _inputs(P=2000, lo=-1.6, hi=1.6)
    keep = _away_from_kinks(grid, (7, 6, 5))
    assert keep.float().mean() > 0.95
    out, mag = R.forward(vol, grid)
    v = vol.clone().requires_grad_(True)
    g = grid.clone().requires_grad_(True)
    ref = _torch_sample(v, g)
    assert R.bar_ratio(out, ref.detach(), mag) <= R.BAR[torch.float64]
    ti, tg = torch.autograd.grad(ref, (v, g), go)
    (gi, gim), (gg, ggm) = R.backward(vol, grid, go)
    assert R.bar_ratio(gi, ti, gim) <= R.BAR[torch.float64]
    assert R.bar_ratio(gg[keep], tg[keep], ggm[keep]) <= R.BAR[torch.float64]
    beyond = (grid.abs() > 1).any(-1)                   # the border clip and its zero gradient are exercised
    assert beyond[keep].float().mean() > 0.3


def test_gradcheck_and_gradgradcheck_away_from_kinks():
    vol, grid, go, _, _ = _inputs(N=2, C=2, D=4, H=3, W=5, P=12)
    grid = grid[:, _away_from_kinks(grid, (5, 3, 4)).all(0)]
    assert grid.shape[1] >= 8
    v = vol.clone().requires_grad_(True)
    g = grid.clone().requires_grad_(True)
    assert torch.autograd.gradcheck(R.sample, (v, g))
    assert torch.autograd.gradgradcheck(R.sample, (v, g))


def test_dbackward_is_the_vjp_of_backward():
    """dbackward's three outputs against autograd of backward's own graph (a float64 central difference of
    <backward, cotangents> in each input would do the same)."""
    vol, grid, go, ggi, ggg = _inputs(P=64)
    v, g, o = (t.clone().requires_grad_(True) for t in (vol, grid, go))
    gi, gg = torch.autograd.grad(R.sample(v, g), (v, g), o, create_graph=True)
    s = (gi * ggi).sum() + (gg * ggg).sum()
    want = torch.autograd.grad(s, (v, g, o))
    got = R.dbackward(ggi, ggg, vol, grid, go)
    for (a, mag), b in zip(got, want):
        assert R.bar_ratio(a, b, mag) <= R.BAR[torch.float64]
    # mag bounds every value
    for a, mag in got:
        assert bool((a.abs() <= mag * (1 + 1e-12)).all())


def test_constant_volume_has_zero_grid_gradient():
    vol, grid, go, _, _ = _inputs(P=500)
    vol = torch.full_like(vol, 0.37)
    (_, _), (gg, mag) = R.backward(vol, grid, go)
    assert float(gg.abs().max()) <= 1e-15 * float(mag.max())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_volume_linear_in_x(dtype):
    """v = a * i + b along x: grad_grid_x = a * W / 2 strictly inside, exactly 0 at and beyond the border; the
    y and z gradients are 0."""
    W, H, D, a = 9, 4, 3, 0.75
    vol = (a * torch.arange(W, dtype=torch.float64) - 2.0).view(1, 1, 1, 1, W).expand(1, 1, D, H, W).contiguous()
    t = R.ties(W, dtype)
    edge = torch.cat([t[0][0], t[0][1], t[W - 1][0], t[W - 1][1]])
    gx = torch.cat([torch.linspace(-1.5, 1.5, 301, dtype=torch.float64).to(dtype), edge])
    grid = torch.stack([gx, torch.zeros_like(gx) + 0.1, torch.zeros_like(gx) - 0.2], -1).unsqueeze(0)
    (_, _), (gg, _) = R.backward(vol.to(dtype), grid, torch.ones(1, 1, gx.numel(), dtype=dtype))
    x = R.unnormalise(gx, W).double()
    inside = (x > 0) & (x < W - 1)
    assert bool(inside.any()) and bool((~inside).any())
    torch.testing.assert_close(gg[0, inside, 0], torch.full_like(gg[0, inside, 0], a * W / 2), rtol=1e-14, atol=0)
    assert bool((gg[0, ~inside, 0] == 0).all()) and bool((gg[0, :, 1:] == 0).all())


def test_size_one_axis_has_zero_gradient_along_it():
    vol, grid, go, ggi, ggg = _inputs(D=1, P=200)
    (_, _), (gg, _) = R.backward(vol, grid, go)
    assert bool((gg[..., 2] == 0).all()) and float(gg[..., :2].abs().max()) > 0
    (_, _), (gg2, _), (_, _) = R.dbackward(ggi, ggg, vol, grid, go)
    assert bool((gg2[..., 2] == 0).all())


def test_tie_sets_are_found_on_every_axis():
    for dtype in (torch.float32, torch.float64):
        for size in (1, 2, 5, 7, 65, 129, 225):
            t = R.ties(size, dtype)
            assert sum(on.numel() for on, _ in t.values()) > 0, (size, dtype)
            for k, (on, flip) in t.items():
                x = R.unnormalise(on, size)
                assert bool((x == k).all())
                xf = R.unnormalise(flip, size)
                assert (bool(xf[0] <= 0) and bool(xf[1] > 0)) if k == 0 else (bool(xf[0] < k) and bool(xf[1] >= k))


# ---- negative controls: each variant must fail a bar the device is held to --------------------------------------
def _axis_no_mask(g, size):
    x, i0, mult = _AXIS(g, size)
    return x, i0, torch.ones_like(mult)


def _axis_half_split(g, size):
    """The 0.5 / 0.5 split of a min / max clip at a tie, the CPU shim's rule."""
    x, i0, mult = _AXIS(g, size)
    xu = R.unnormalise(g, size).double()
    return x, i0, torch.where((xu == 0) | (xu == size - 1), torch.full_like(mult, 0.5), mult)


def _axis_round(g, size):
    x, i0, mult = _AXIS(g, size)
    return x, torch.round(x).long(), mult


def _unnormalise_align_corners(g, size):
    return ((g.double() + 1) / 2 * (size - 1)).to(g.dtype)


def _unnormalise_f64(g, size):
    return ((g.double() + 1) * size - 1) / 2


_AXIS = R._axis


def _tie_inputs(dtype, sizes=(7, 6, 5), seed=1):
    """A grid whose every axis takes its tie values (exact hits, their ulp neighbours and the flip pairs)."""
    gen = torch.Generator().manual_seed(seed)
    cols = []
    for s in sizes:
        vals = torch.cat([torch.cat([on, R.ulp_neighbours(on), flip]) if on.numel() else flip
                          for on, flip in R.ties(s, dtype).values()])
        cols.append(vals[torch.randint(0, vals.numel(), (400,), generator=gen)])
    vol, _, go, ggi, ggg = _inputs(P=400, dtype=dtype, N=1, seed=seed)
    return vol, torch.stack(cols, -1).unsqueeze(0), go, ggi, ggg


@pytest.mark.parametrize("name", ["no_mask", "half_split", "align_corners", "round", "x_in_float64"])
def test_negative_controls_fail_the_bars(name, monkeypatch):
    dtype = torch.float32 if name == "x_in_float64" else torch.float64
    vol, grid, go, ggi, ggg = _tie_inputs(dtype)
    rnd = _inputs(N=1, P=400, lo=-1.6, hi=1.6, dtype=dtype, seed=2)[1]
    grid = torch.cat([grid, rnd], dim=1)
    go, ggg = torch.cat([go, go], -1), torch.cat([ggg, ggg], 1)
    correct = _all_outputs(vol, grid, go, ggi, ggg)
    masks = _masks(vol, grid)
    patch = {"no_mask": ("_axis", _axis_no_mask), "half_split": ("_axis", _axis_half_split),
             "round": ("_axis", _axis_round), "align_corners": ("unnormalise", _unnormalise_align_corners),
             "x_in_float64": ("unnormalise", _unnormalise_f64)}[name]
    monkeypatch.setattr(R, *patch)
    failed = _fails(_all_outputs(vol, grid, go, ggi, ggg), correct, dtype, masks)
    print("%s fails: %s" % (name, failed))
    must = {"no_mask": ("zero", "bwd_grid"), "half_split": ("bwd_grid", "dbwd_grid"),
            "align_corners": ("fwd", "index"), "round": ("fwd", "index"), "x_in_float64": ("index",)}[name]
    assert all(k in failed for k in must), failed


def test_half_split_needs_the_ties():
    """The shim's rule passes every bar on random points: only the constructed ties expose it.  (Computing x in
    float64 for float32 grids fails the value bars even there, by the rounding of x.)"""
    vol, grid, go, ggi, ggg = _inputs(N=1, P=400, seed=3)
    correct = _all_outputs(vol, grid, go, ggi, ggg)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(R, "_axis", _axis_half_split)
        assert _fails(_all_outputs(vol, grid, go, ggi, ggg), correct, torch.float64, _masks(vol, grid)) == {}
