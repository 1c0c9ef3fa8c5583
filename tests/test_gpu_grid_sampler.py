"""GPU: the trilinear sampler (csrc/grid_sampler.cu) through ops.grid_sample3d_* and the raw C ABI, float32 and
float64, against the float64 restatement tests/grid_sampler_ref.py (pinned on CPU by test_grid_sampler_ref_cpu.py).

Geometries: the production skin-weight volume (24 x 65 x 225 x 129, synth.make_skinner), 5 x 1 x 2 x 7 (size-1 and
size-2 axes), N = 3 with distinct volumes and grids, C = 1 and C = 33.  Points: random in and beyond [-1.2, 1.2];
points whose kernel x is exactly an integer (0 and size - 1 included where representable), one ulp either side of
each, and the pairs between which floor or the mask flips; 200 000 points in one cell (grad_input by atomics);
270 336 + 1 000 points, one more than a grid-stride wave.  Layouts: channels-last and sliced volumes.

Bars: corner indices bit-exact; grad_grid exactly 0 wherever the mask is 0; |a - b| <= c * mag elementwise (mag the
float64 sum of |terms|), c = 1e-6 for float32 and 1e-13 for float64.  The measured maxima are printed."""
import ctypes as C
import importlib
import sys
import types

import pytest
import torch

import grid_sampler_ref as R

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.float64]
WAVE = 132 * 16 * 128          # the sampler's grid-stride launch covers this many points per pass
_MAX = {}                      # (dtype, output) -> largest |a - b| / mag seen


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for (dt, name), r in sorted(_MAX.items(), key=lambda kv: (str(kv[0][0]), kv[0][1])):
        print("grid sampler %s %-10s max |a-b|/mag %.2e (bar %.0e)" % (str(dt)[6:], name, r, R.BAR[dt]))


def _ops():
    from selfreconcode_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _grid(N, P, gen, dtype, lo=-1.2, hi=1.2):
    return (lo + (hi - lo) * torch.rand(N, 1, 1, P, 3, generator=gen, dtype=torch.float64)).to(dtype)


def _tie_grid(N, sizes, dtype, gen, P=None):
    """[N,1,1,P,3]: every axis drawn from its tie values (exact integer x, their ulp neighbours, the flip pairs),
    or, for a third of the entries, uniform in [-1.2, 1.2].  Asserts that every axis has exact hits."""
    cols = []
    for s in sizes:
        t = R.ties(s, dtype)
        on = torch.cat([o for o, _ in t.values()])
        assert on.numel() > 0, "no grid value puts x exactly on an integer of an axis of %d" % s
        vals = torch.cat([on, R.ulp_neighbours(on)] + [f for _, f in t.values()])
        P = P or 3 * vals.numel()
        col = vals[torch.randint(0, vals.numel(), (N, P), generator=gen)]
        rnd = _grid(N, P, gen, dtype)[:, 0, 0, :, 0]
        cols.append(torch.where(torch.rand(N, P, generator=gen) < 1 / 3, rnd, col))
    return torch.stack(cols, -1).view(N, 1, 1, -1, 3)


def _cotangents(vol, grid, gen):
    N, Cc = vol.shape[:2]
    P = grid.shape[3]
    rn = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64).to(vol.dtype)
    return rn(N, Cc, 1, 1, P), rn(*vol.shape), rn(*grid.shape)


def _record(dt, name, a, b, mag):
    r = R.bar_ratio(a, b, mag)
    _MAX[(dt, name)] = max(_MAX.get((dt, name), 0.0), r)
    assert r <= R.BAR[dt], "%s %s: max |a-b|/mag %.3e > %.0e" % (dt, name, r, R.BAR[dt])


def _device(vol, grid, go, ggi, ggg):
    ops = _ops()
    out, cidx = ops.grid_sample3d_forward(vol, grid, want_corner_idx=True)
    gi, gg = ops.grid_sample3d_backward(vol, grid, go)
    di, dg, dgo = ops.grid_sample3d_dbackward(ggi, ggg, vol, grid, go)
    return {"fwd": out, "cidx": cidx, "bwd_input": gi, "bwd_grid": gg, "dbwd_input": di, "dbwd_grid": dg,
            "dbwd_gout": dgo}


def _check(vol, grid, go, ggi, ggg, dev=None, rows=None):
    """Runs the three kernels (unless `dev` holds their outputs) and holds them to the bars; `rows` (a slice of the
    flattened N*P points) selects the per-point rows that are compared.  Returns the device outputs."""
    dev = dev or _device(vol, grid, go, ggi, ggg)
    dt, (N, Cc, D, H, W) = vol.dtype, vol.shape
    rows = rows or slice(None)
    pt = lambda t, c: t.reshape(N, c, -1).transpose(1, 2).reshape(-1, c)[rows]     # [N*P rows, c]
    g3 = grid.reshape(N, -1, 3)
    assert torch.equal(dev["cidx"].reshape(-1, 3)[rows], R.corner_index(vol, g3).reshape(-1, 3)[rows].to(vol.device))
    mask = torch.stack([a[2] for a in R.axes(g3, (W, H, D))], -1).reshape(-1, 3)[rows]
    for name in ("bwd_grid", "dbwd_grid"):
        assert bool((dev[name].reshape(-1, 3)[rows][mask == 0] == 0).all()), name + " is not 0 where the mask is 0"
    out, mag = R.forward(vol, g3)
    _record(dt, "fwd", pt(dev["fwd"], Cc), pt(out, Cc), pt(mag, Cc))
    (gi, gim), (gg, ggm) = R.backward(vol, g3, go)
    _record(dt, "bwd_input", dev["bwd_input"], gi, gim)
    _record(dt, "bwd_grid", dev["bwd_grid"].reshape(-1, 3)[rows], gg.reshape(-1, 3)[rows], ggm.reshape(-1, 3)[rows])
    (di, dim), (dg, dgm), (dgo, dgom) = R.dbackward(ggi, ggg, vol, g3, go)
    _record(dt, "dbwd_input", dev["dbwd_input"], di, dim)
    _record(dt, "dbwd_grid", dev["dbwd_grid"].reshape(-1, 3)[rows], dg.reshape(-1, 3)[rows], dgm.reshape(-1, 3)[rows])
    _record(dt, "dbwd_gout", pt(dev["dbwd_gout"], Cc), pt(dgo, Cc), pt(dgom, Cc))
    return dev


# ---- geometries ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def production_volume(cuda_dev):
    from selfreconcode_b200 import synth
    ws = synth.make_skinner().ws
    assert tuple(ws.shape) == (1, 24, 65, 225, 129)
    return ws.to(cuda_dev)


@pytest.mark.parametrize("dtype", DTYPES)
def test_production_volume(production_volume, dtype, cuda_dev):
    gen = _gen(1)
    vol = production_volume.to(dtype)
    grid = torch.cat([_grid(1, 6000, gen, dtype), _grid(1, 2000, gen, dtype, -3.0, 3.0),
                      _tie_grid(1, (129, 225, 65), dtype, gen, P=4000)], dim=3).to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(vol, grid, gen))
    _check(vol, grid, go, ggi, ggg)


@pytest.mark.parametrize("dtype", DTYPES)
def test_size_one_and_two_axes(dtype, cuda_dev):
    gen = _gen(2)
    vol = torch.randn(1, 5, 1, 2, 7, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    grid = torch.cat([_grid(1, 500, gen, dtype, -1.6, 1.6), _tie_grid(1, (7, 2, 1), dtype, gen)], 3).to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(vol, grid, gen))
    dev = _check(vol, grid, go, ggi, ggg)
    assert bool((dev["bwd_grid"][..., 2] == 0).all()) and bool((dev["dbwd_grid"][..., 2] == 0).all())


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_of_three(dtype, cuda_dev):
    """Distinct volumes and grids per batch entry; each entry equals its own N = 1 launch (bit-exact where no
    atomics are involved)."""
    gen = _gen(3)
    vol = torch.randn(3, 4, 6, 5, 9, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    grid = torch.cat([_grid(3, 700, gen, dtype), _tie_grid(3, (9, 5, 6), dtype, gen, P=600)], 3).to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(vol, grid, gen))
    dev = _check(vol, grid, go, ggi, ggg)
    for n in range(3):
        one = _device(vol[n:n + 1], grid[n:n + 1], go[n:n + 1], ggi[n:n + 1], ggg[n:n + 1])
        for name in ("fwd", "cidx", "bwd_grid", "dbwd_grid", "dbwd_gout"):
            assert torch.equal(one[name], dev[name][n:n + 1]), (n, name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("channels", [1, 33])
def test_channel_counts(channels, dtype, cuda_dev):
    gen = _gen(4 + channels)
    vol = torch.rand(2, channels, 7, 11, 13, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    grid = torch.cat([_grid(2, 1500, gen, dtype), _tie_grid(2, (13, 11, 7), dtype, gen, P=500)], 3).to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(vol, grid, gen))
    _check(vol, grid, go, ggi, ggg)


@pytest.mark.parametrize("dtype", DTYPES)
def test_many_points_in_one_cell(dtype, cuda_dev):
    """200 000 points inside cell (4, 3, 2) of a 9 x 7 x 6 volume: the eight corners' grad_input are sums of
    200 000 atomically added terms."""
    gen = _gen(5)
    W, H, D, P = 9, 7, 6, 200_000
    vol = torch.randn(1, 3, D, H, W, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    x = torch.tensor([4.0, 3.0, 2.0], dtype=torch.float64) + 0.02 + 0.96 * torch.rand(P, 3, generator=gen,
                                                                                          dtype=torch.float64)
    size = torch.tensor([W, H, D], dtype=torch.float64)
    grid = ((2 * x + 1) / size - 1).to(dtype).view(1, 1, 1, P, 3).to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(vol, grid, gen))
    dev = _check(vol, grid, go, ggi, ggg)
    assert bool((dev["cidx"].view(-1, 3).cpu() == torch.tensor([4, 3, 2], dtype=torch.int32)).all())
    touched = torch.zeros(D, H, W, dtype=torch.bool)
    touched[2:4, 3:5, 4:6] = True
    for name in ("bwd_input", "dbwd_input"):
        assert bool((dev[name][0][:, ~touched.to(cuda_dev)] == 0).all()), name


@pytest.mark.parametrize("dtype", DTYPES)
def test_second_grid_stride_wave(dtype, cuda_dev):
    """270 336 + 1 000 points: the last 1 000 are a second pass of the grid-stride loop.  Outputs are launched into
    NaN-filled buffers through the C ABI, so a row the second pass missed stays NaN."""
    gen = _gen(6)
    P = WAVE + 1000
    vol = torch.rand(1, 4, 5, 8, 6, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    grid = _grid(1, P, gen, dtype).to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(vol, grid, gen))
    dev = _abi_all(vol, grid, go, ggi, ggg)
    for name, t in dev.items():
        assert not bool(torch.isnan(t.double()).any()), name
    _check(vol, grid, go, ggi, ggg, dev=dev, rows=slice(WAVE, None))
    _check(vol, grid, go, ggi, ggg, dev=dev)


# ---- layouts --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_channels_last_and_sliced_volumes(dtype, cuda_dev):
    """The kernels read the volume through its strides (and write grad_input contiguous): a channels-last permute
    and a sliced view give the contiguous volume's results (bit-exact where no atomics are involved)."""
    gen = _gen(7)
    N, Cc, D, H, W = 2, 5, 6, 7, 9
    base = torch.randn(N, Cc, D, H, W, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    cl = base.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3)
    big = torch.randn(N, Cc + 2, D + 1, H, 2 * W, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    big[:, 1:Cc + 1, 1:, :, ::2] = base
    sliced = big[:, 1:Cc + 1, 1:, :, ::2]
    assert not cl.is_contiguous() and not sliced.is_contiguous()
    grid = torch.cat([_grid(N, 800, gen, dtype, -1.3, 1.3), _tie_grid(N, (W, H, D), dtype, gen, P=400)], 3)
    grid = grid.to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(base, grid, gen))
    want = _device(base, grid, go, ggi, ggg)
    for vol in (cl, sliced):
        dev = _check(vol, grid, go, ggi, ggg)
        for name in ("fwd", "cidx", "bwd_grid", "dbwd_grid", "dbwd_gout"):
            assert torch.equal(dev[name], want[name]), name
        assert dev["bwd_input"].is_contiguous() and dev["dbwd_input"].is_contiguous()


# ---- non-finite coordinates --------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_non_finite_coordinates(dtype, cuda_dev):
    """NaN is sampled at 0 with mask 0 (its backward is the gradient of what the forward computed); +-inf clip to
    the ends.  Every output stays finite."""
    gen = _gen(8)
    vol = torch.randn(1, 3, 4, 5, 6, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    grid = _grid(1, 300, gen, dtype)
    special = torch.tensor([float("nan"), float("inf"), -float("inf")], dtype=dtype)
    grid.view(-1)[::2] = special[torch.randint(0, 3, (grid.numel() // 2 + grid.numel() % 2,), generator=gen)]
    grid = grid.to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(vol, grid, gen))
    dev = _check(vol, grid, go, ggi, ggg)
    for name, t in dev.items():
        assert bool(torch.isfinite(t.double()).all()), name


# ---- the C ABI: sentinels and status codes -----------------------------------------------------------------------
def _abi(kind, dtype):
    from selfreconcode_b200 import _lib
    return getattr(_lib.load(), "sr_grid_sample3d_%s_%s" % (kind, {torch.float32: "f32", torch.float64: "f64"}[dtype]))


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _istr(t):
    return (C.c_int64 * 5)(*t.stride())


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _abi_all(vol, grid, go, ggi, ggg):
    """The three kernels through the C ABI with every output but grad_input NaN-filled (corner indices -7) and
    grad_input zeroed, as the atomics require."""
    dt, (N, Cc, D, H, W), P = vol.dtype, vol.shape, grid.shape[3]
    nan = lambda *s: torch.full(s, float("nan"), dtype=dt, device=vol.device)
    out, gg, dg, dgo = nan(N, Cc, 1, 1, P), nan(N, 1, 1, P, 3), nan(N, 1, 1, P, 3), nan(N, Cc, 1, 1, P)
    cidx = torch.full((N, P, 3), -7, dtype=torch.int32, device=vol.device)
    gi, di = torch.zeros_like(vol).contiguous(), torch.zeros_like(vol).contiguous()
    g, o, q, qq = grid.contiguous(), go.contiguous(), ggi.contiguous(), ggg.contiguous()
    assert _abi("fwd", dt)(_p(vol), _istr(vol), _p(g), _p(out), _p(cidx), N, Cc, D, H, W, P, _s()) == 0
    assert _abi("bwd", dt)(_p(vol), _istr(vol), _p(g), _p(o), _p(gi), _p(gg), N, Cc, D, H, W, P, _s()) == 0
    assert _abi("dbwd", dt)(_p(q), _p(qq), _p(vol), _istr(vol), _p(g), _p(o), _p(di), _p(dg), _p(dgo),
                            N, Cc, D, H, W, P, _s()) == 0
    torch.cuda.synchronize()
    return {"fwd": out, "cidx": cidx, "bwd_input": gi, "bwd_grid": gg, "dbwd_input": di, "dbwd_grid": dg,
            "dbwd_gout": dgo}


@pytest.mark.parametrize("dtype", DTYPES)
def test_c_abi_fills_every_output(dtype, cuda_dev):
    gen = _gen(9)
    vol = torch.randn(2, 3, 4, 6, 5, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    grid = torch.cat([_grid(2, 400, gen, dtype, -1.5, 1.5), _tie_grid(2, (5, 6, 4), dtype, gen, P=300)], 3)
    grid = grid.to(cuda_dev)
    go, ggi, ggg = (t.to(cuda_dev) for t in _cotangents(vol, grid, gen))
    dev = _abi_all(vol, grid, go, ggi, ggg)
    for name, t in dev.items():
        assert not bool(torch.isnan(t.double()).any()), name
    _check(vol, grid, go, ggi, ggg, dev=dev)


@pytest.mark.parametrize("dtype", DTYPES)
def test_c_abi_status_codes(dtype, cuda_dev):
    from selfreconcode_b200._lib import SR_EINVAL, SR_OK
    N, Cc, D, H, W, P = 1, 2, 3, 4, 5, 16
    t = lambda *s: torch.zeros(*s, dtype=dtype, device=cuda_dev)
    vol, grid, go, gi, gg = t(N, Cc, D, H, W), t(N, P, 3), t(N, Cc, P), t(N, Cc, D, H, W), t(N, P, 3)
    out, ggo = t(N, Cc, P), t(N, Cc, P)
    cidx = torch.full((N, P, 3), -7, dtype=torch.int32, device=cuda_dev)
    fwd, bwd, dbwd = _abi("fwd", dtype), _abi("bwd", dtype), _abi("dbwd", dtype)

    def call(kind, n=N, c=Cc, d=D, h=H, w=W, p=P, istr=True, **null):
        a = {"vol": vol, "grid": grid, "go": go, "gi": gi, "gg": gg, "out": out, "ggo": ggo, "cidx": cidx,
             "ggi": gi, "ggg": gg}
        a.update({k: None for k in null})
        st = _istr(vol) if istr else None
        if kind == "fwd":
            return fwd(_p(a["vol"]), st, _p(a["grid"]), _p(a["out"]), _p(a["cidx"]), n, c, d, h, w, p, _s())
        if kind == "bwd":
            return bwd(_p(a["vol"]), st, _p(a["grid"]), _p(a["go"]), _p(a["gi"]), _p(a["gg"]), n, c, d, h, w, p, _s())
        return dbwd(_p(a["ggi"]), _p(a["ggg"]), _p(a["vol"]), st, _p(a["grid"]), _p(a["go"]), _p(a["gi"]),
                    _p(a["gg"]), _p(a["ggo"]), n, c, d, h, w, p, _s())

    for kind in ("fwd", "bwd", "dbwd"):
        assert call(kind) == SR_OK
        assert call(kind, p=0) == SR_OK and call(kind, n=0) == SR_OK
        for bad in ({"d": 0}, {"h": 0}, {"w": -1}, {"c": -1}, {"p": -1}, {"istr": False}, {"grid": 1}):
            assert call(kind, **bad) == SR_EINVAL, (kind, bad)
    for kind, ptrs in (("fwd", ("vol", "out")), ("bwd", ("vol", "go", "gi", "gg")),
                       ("dbwd", ("ggi", "ggg", "vol", "go", "gi", "gg", "ggo"))):
        for name in ptrs:
            assert call(kind, **{name: 1}) == SR_EINVAL, (kind, name)
    # C = 0: the channel arrays may be null; corner indices and the (zero) grid gradient are still written
    gg.fill_(float("nan"))
    assert call("fwd", c=0, vol=1, out=1) == SR_OK
    assert call("bwd", c=0, vol=1, go=1, gi=1) == SR_OK
    torch.cuda.synchronize()
    assert bool((cidx >= 0).all()) and bool((gg == 0).all())
    gg.fill_(float("nan"))
    assert call("dbwd", c=0, vol=1, go=1, gi=1, ggi=1, ggo=1) == SR_OK
    torch.cuda.synchronize()
    assert bool((gg == 0).all())


@pytest.mark.parametrize("dtype", DTYPES)
def test_ops_empty_and_zero_channel_calls(dtype, cuda_dev):
    ops = _ops()
    gen = _gen(10)
    grid = _grid(2, 50, gen, dtype).to(cuda_dev)
    vol0 = torch.zeros(2, 0, 3, 4, 5, dtype=dtype, device=cuda_dev)
    out, cidx = ops.grid_sample3d_forward(vol0, grid, want_corner_idx=True)
    assert out.shape == (2, 0, 1, 1, 50)
    assert torch.equal(cidx.cpu(), R.corner_index(vol0.cpu(), grid.cpu()))
    gi, gg = ops.grid_sample3d_backward(vol0, grid, torch.zeros(2, 0, 1, 1, 50, dtype=dtype, device=cuda_dev))
    assert gi.shape == vol0.shape and bool((gg == 0).all())
    di, dg, dgo = ops.grid_sample3d_dbackward(vol0, torch.randn(grid.shape, generator=gen).to(grid), vol0, grid,
                                              torch.zeros(2, 0, 1, 1, 50, dtype=dtype, device=cuda_dev))
    assert di.shape == vol0.shape and bool((dg == 0).all()) and dgo.shape == (2, 0, 1, 1, 50)
    vol = torch.randn(2, 3, 3, 4, 5, generator=gen, dtype=torch.float64).to(dtype).to(cuda_dev)
    empty = grid[:, :, :, :0]
    assert ops.grid_sample3d_forward(vol, empty).shape == (2, 3, 1, 1, 0)
    gi, gg = ops.grid_sample3d_backward(vol, empty, torch.zeros(2, 3, 1, 1, 0, dtype=dtype, device=cuda_dev))
    assert bool((gi == 0).all()) and gg.shape == empty.shape


def test_ops_refuse_mismatched_arguments(cuda_dev):
    ops = _ops()
    vol = torch.rand(2, 3, 4, 5, 6, device=cuda_dev)
    grid = torch.rand(2, 1, 1, 10, 3, device=cuda_dev)
    go = torch.rand(2, 3, 1, 1, 10, device=cuda_dev)
    with pytest.raises(RuntimeError, match="float32"):
        ops.grid_sample3d_forward(vol, grid.double())
    with pytest.raises(RuntimeError, match="batch sizes"):
        ops.grid_sample3d_forward(vol, grid[:1])
    with pytest.raises(RuntimeError, match="float32"):
        ops.grid_sample3d_backward(vol, grid, go.double())
    with pytest.raises(RuntimeError, match="gg_input"):
        ops.grid_sample3d_dbackward(vol[:, :2], grid, vol, grid, go)
    with pytest.raises(RuntimeError, match="grid"):
        ops.grid_sample3d_forward(vol, grid[..., :2])


# ---- end to end through autograd ---------------------------------------------------------------------------------
def _restatement_backend(seen):
    """A `GridSamplerMine` module computed by the restatement (float64, on the tensors' device), recording whether
    each cotangent arrived contiguous."""
    m = types.ModuleType("GridSamplerMine")

    def forward(vol, grid, interp=0, pad=1):
        N, Cc = vol.shape[:2]
        return R.forward(vol, grid)[0].to(vol.dtype).view((N, Cc) + tuple(grid.shape[1:4]))

    def backward(vol, grid, go, interp=0, pad=1):
        seen.append(go.is_contiguous())
        (gi, _), (gg, _) = R.backward(vol, grid, go)
        return gi.to(vol.dtype), gg.to(vol.dtype).view(grid.shape)

    def dbackward(ggi, ggg, vol, grid, go, interp=0, pad=1):
        (di, _), (dg, _), (dgo, _) = R.dbackward(ggi, ggg, vol, grid, go)
        return di.to(vol.dtype), dg.to(vol.dtype).view(grid.shape), dgo.to(vol.dtype).view(go.shape)

    m.forward, m.backward, m.dbackward = forward, backward, dbackward
    return m


def _skinned_loss(sk, pts, conds, w):
    """Mesh-mode skinning, then a loss on d(skinned points . w)/d(points): backpropagating it runs the sampler's
    second-order backward (_SampleVjp.backward)."""
    p = pts.clone().requires_grad_(True)
    y = sk(p, conds)
    (gp,) = torch.autograd.grad((y * w).sum(), p, create_graph=True)
    loss = (gp * gp).sum() + (y * y).sum()
    loss.backward()
    return loss.detach(), p.grad


def test_skinning_loss_through_second_order_matches_float64(cuda_dev, monkeypatch):
    """The skinner on the kernels (float32 and float64 entry points) and on the restatement as its sampler backend,
    in float32 and float64 modules, against the float64 module on the restatement (the twin).  float64 kernels vs
    the twin isolate the sampler.  The skin weights sum to 1, so their point gradients cancel across the 24
    channels: a kernel's error scales with the sum of |terms| (the bars above), not with d/dpoints itself, and the
    float32 kernels' d/dpoints error is that of the float64 kernels scaled by the two unit roundoffs -- not the
    float32 module's on the restatement, which rounds only the sampler's results."""
    from helpers import dropin, elem_err
    dropin()
    from selfreconcode_b200 import synth
    gen = _gen(11)
    poses, trans, _ = synth.make_frame_params(12, 2)
    lo, hi = torch.tensor(synth.B_MIN), torch.tensor(synth.B_MAX)
    # mesh-mode points [frames, V, 3], a tenth of them outside the box on some axis (clipped, mask 0)
    pts = lo + (hi - lo) * (-0.05 + 1.1 * torch.rand(2, 3000, 3, generator=gen))
    w = torch.randn(2, 3000, 3, generator=gen)
    kernels = importlib.import_module("GridSamplerMine")
    res, seen = {}, []
    for dtype in (torch.float32, torch.float64):
        sk = synth.make_skinner().to(cuda_dev).to(dtype)
        for backend in ("kernels", "restatement"):
            monkeypatch.setitem(sys.modules, "GridSamplerMine",
                                kernels if backend == "kernels" else _restatement_backend(seen))
            ps = poses.to(cuda_dev, dtype).requires_grad_(True)
            loss, gp = _skinned_loss(sk, pts.to(cuda_dev, dtype), [ps, trans.to(cuda_dev, dtype)],
                                     w.to(cuda_dev, dtype))
            res[(dtype, backend)] = [loss.reshape(1), gp, ps.grad]
    assert seen and not all(seen), "some cotangent should arrive non-contiguous (the skinner passes a transposed view)"
    twin = res[(torch.float64, "restatement")]
    err = {k: [elem_err(a.cpu(), b.cpu()) for a, b in zip(v, twin)] for k, v in res.items() if v is not twin}
    for k, e in err.items():
        print("skinning loss through the second order, %s %s vs the float64 twin: loss %.1e, d/dpoints %.1e, "
              "d/dposes %.1e (elem_err)" % (str(k[0])[6:], k[1], *e))
    assert max(err[(torch.float64, "kernels")]) < 1e-9
    assert max(err[(torch.float32, "restatement")]) < 1e-4
    el, ep, epose = err[(torch.float32, "kernels")]
    assert el < 1e-5 and epose < 1e-4 and ep < 1e-2
