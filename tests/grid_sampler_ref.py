"""float64 restatement of the trilinear grid sampler of csrc/grid_sampler.cu (border padding, align_corners=False):
forward, first-order backward and second-order backward, written from the sampler's definition.

* The un-normalised coordinate x follows the kernel's rule for the grid's dtype (`unnormalise`), so corner indices
  and border decisions are the kernel's own even where x lies exactly on a voxel face.
* floor(x) and the border mask (1 strictly inside (0, size-1); 0 at or beyond either end, and for NaN) are taken
  from that x and held constant.  Everything after them -- the corner weights, the corners beyond the volume and the
  size/2 * mask chain factor -- is differentiable float64 torch, so the first and second order come from
  torch.autograd.
* Every output comes with `mag`, the float64 sum of the absolute values of the terms it is a sum of; the device bars
  are |a - b| <= c * mag.  It is the same computation on |inputs| with d(weight towards i0)/dx taken as +1 instead
  of -1, so that every term is a product of non-negative factors.

Volumes are [N,C,D,H,W], grids [N,...,3] (x, y, z), per-point outputs [N,C,P] and [N,P,3] with P the grid's points.
Works on CPU or CUDA tensors.  `_axis` is the one place that decides x, floor(x) and the mask; the negative controls
of test_grid_sampler_ref_cpu.py substitute it."""
import torch


def unnormalise(g, size):
    """The kernel's x for grid values g on an axis of `size` voxels, in g's dtype.  float32:
    fl32((double(fl32(fl32(g + 1) * size)) - 1) / 2); float64: ((g + 1) * size - 1) / 2."""
    if g.dtype == torch.float32:
        return (((g + 1) * size).double() - 1).div(2).float()
    if g.dtype == torch.float64:
        return ((g + 1) * size - 1) / 2
    raise TypeError("the sampler takes float32 or float64 grids, not %s" % g.dtype)


def _axis(g, size):
    """(x, i0, mult) for grid values g: the clipped coordinate (float64), floor(x) (int64) and the border mask
    (float64, 0 or 1)."""
    x = unnormalise(g, size).double()
    mult = ((x > 0) & (x < size - 1)).double()
    x = torch.where(x > 0, x, torch.zeros_like(x)).clamp(max=size - 1)
    return x, torch.floor(x).long(), mult


def axes(grid, sizes):
    """[(x, i0, mult)] of the three axes of grid [N,P,3]; sizes = (W, H, D)."""
    g = grid.detach()
    return [_axis(g[..., k], s) for k, s in enumerate(sizes)]


def corner_index(vol, grid):
    """[N,P,3] int32: floor of the clipped x, y, z -- the kernel's corner indices."""
    N, _, D, H, W = vol.shape
    return torch.stack([a[1] for a in axes(grid.reshape(N, -1, 3), (W, H, D))], dim=-1).int()


def sample(vol, grid, magnitude=False, rule_grid=None):
    """out [N,C,P] in float64, differentiable in vol and grid.  x, floor(x) and the mask come from `rule_grid` (same
    values as grid, in the dtype whose rule applies; default grid itself).  magnitude=True gives the `mag` of the
    module docstring for inputs that are already non-negative."""
    N, C, D, H, W = vol.shape
    gd = grid.reshape(N, -1, 3).double()
    P = gd.shape[1]
    ax = axes((grid if rule_grid is None else rule_grid).reshape(N, -1, 3), (W, H, D))
    a = []
    for k, ((x, i0, mult), size) in enumerate(zip(ax, (W, H, D))):
        t = gd[..., k]
        # value 0, slope size/2 * mult; the where keeps a non-finite t out of the value and the gradients
        u = torch.where(mult != 0, (t - t.detach()) * (mult * (size / 2)), torch.zeros_like(t))
        a.append(((i0 + 1) - x + (u if magnitude else -u), (x - i0) + u))
    flat = vol.double().reshape(N, C, D * H * W)
    i0x, i0y, i0z = (q[1] for q in ax)
    out = flat.new_zeros((N, C, P))
    for bz in (0, 1):
        for by in (0, 1):
            for bx in (0, 1):
                ix, iy, iz = i0x + bx, i0y + by, i0z + bz
                ok = ((ix < W) & (iy < H) & (iz < D)).double()
                lin = (iz.clamp(max=D - 1) * H + iy.clamp(max=H - 1)) * W + ix.clamp(max=W - 1)
                v = torch.gather(flat, 2, lin.unsqueeze(1).expand(N, C, P))
                w = a[0][bx] * a[1][by] * a[2][bz] * ok
                out = out + v * w.unsqueeze(1)
    return out


def _in(t, magnitude, grad=True):
    t = t.detach().double()
    return (t.abs() if magnitude else t).requires_grad_(grad)


def _zero_if_none(t, like):
    return torch.zeros_like(like) if t is None else t


def forward(vol, grid):
    """(out, mag) [N,C,P]: the sampled volume; grid's dtype selects the x rule."""
    with torch.no_grad():
        return tuple(sample(_in(vol, m, False), grid, m) for m in (False, True))


def backward(vol, grid, gout):
    """[(d vol, mag) [N,C,D,H,W], (d grid, mag) [N,P,3]]: the VJP of `forward` with cotangent gout [N,C,P]."""
    N, C = vol.shape[:2]
    res = []
    with torch.enable_grad():                                       # also when called from a Function's forward
        for m in (False, True):
            v, g = _in(vol, m), grid.detach().reshape(N, -1, 3).double().requires_grad_(True)
            out = sample(v, g, m, grid)
            res.append(torch.autograd.grad(out, (v, g), _in(gout, m, False).reshape(out.shape)))
    return list(zip(*res))


def dbackward(ggi, ggg, vol, grid, gout):
    """[(d vol, mag), (d grid, mag), (d gout, mag) [N,C,P]]: the VJP of `backward` with cotangents ggi (like vol)
    and ggg (like the grid)."""
    N, C = vol.shape[:2]
    res = []
    with torch.enable_grad():
        for m in (False, True):
            v, g = _in(vol, m), grid.detach().reshape(N, -1, 3).double().requires_grad_(True)
            go = _in(gout, m).reshape(N, C, -1)
            out = sample(v, g, m, grid)
            gi, gg = torch.autograd.grad(out, (v, g), go, create_graph=True)
            s = (gi * _in(ggi, m, False)).sum() + (gg * _in(ggg, m, False).reshape(gg.shape)).sum()
            d = torch.autograd.grad(s, (v, g, go), allow_unused=True)
            res.append([_zero_if_none(x, y).detach() for x, y in zip(d, (v, g, go))])
    return list(zip(*res))


def ties(size, dtype, targets=None, window=1 << 14, keep=16):
    """{k: (on, flip)} for each integer k of `targets` (default: every index of a short axis; 0, 1, 2, size // 2,
    size - 3, size - 2, size - 1 otherwise).  `on` holds the grid values g (dtype) whose kernel x is exactly k, `flip`
    the two consecutive values between which the decision at k changes: x < k to x >= k (floor, and the mask at
    size - 1), x <= 0 to x > 0 at k = 0.  x depends on g only through t = fl(g + 1), so the scan runs over the
    `window` representable values either side of both t = (2k + 1) / size (with g = t - 1) and g itself.  Near k = 0
    there is often no g with x = k: there g + 1 rounds to multiples of ulp(g).  At most `keep` values of `on` are
    kept per k, spread over the ones found."""
    if targets is None:
        targets = range(size) if size <= 8 else sorted({0, 1, 2, size // 2, size - 3, size - 2, size - 1})
    ity = {torch.float32: torch.int32, torch.float64: torch.int64}[dtype]
    steps = torch.arange(-window, window + 1, dtype=ity)
    out = {}
    for k in targets:
        t0 = torch.tensor([(2 * k + 1) / size], dtype=dtype)
        t, g = ((v.view(ity) + steps).view(dtype) for v in (t0, t0 - 1))
        g = torch.cat([t[t > 0] - 1, g])
        g = torch.unique(g[torch.isfinite(g)])                      # sorted, and x is non-decreasing in g
        x = unnormalise(g, size)
        above = x > 0 if k == 0 else x >= k
        j = int(above.int().argmax())
        assert 0 < j and bool(above[j:].all()) and not bool(above[:j].any()), "scan window misses the flip at %d" % k
        on = g[x == k]
        if on.numel() > keep:                                       # around g = 0 every tiny g is a hit
            on = on[torch.linspace(0, on.numel() - 1, keep).long()]
        out[k] = (on, g[j - 1:j + 1])
    return out


def ulp_neighbours(g):
    """The values one ulp below and above each of g (in g's dtype)."""
    return torch.cat([torch.nextafter(g, torch.full_like(g, -float("inf"))),
                      torch.nextafter(g, torch.full_like(g, float("inf")))])


# |a - b| <= BAR[dtype] * mag, elementwise: about 16 roundings per term (8 FMAs and the weight products)
BAR = {torch.float32: 1e-6, torch.float64: 1e-13}


def bar_ratio(a, b, mag):
    """max |a - b| / mag over the elements (0 where both sides are 0; inf where mag is 0 and a != b)."""
    d = (a.double() - b.double()).abs()
    r = torch.where(d == 0, torch.zeros_like(d), d / mag)
    return float(r.max()) if r.numel() else 0.0
