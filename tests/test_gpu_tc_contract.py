"""GPU: the tensor-core layer kernel (tc_sweep_kernel, csrc/tc_gemm.cu) and the weight-gradient / column-sum kernels
(csrc/tc_wgrad.cu) against a plain float64 restatement of their contract.  The kernels are called through the C ABI so
that every sr_tc_linear argument is reachable: the act' stash, the reverse-mode `mul_*` inputs, m_dev, the `out`
window.

  * all 14 layer instantiations (activation x rows per point x forward / reverse) over row counts that leave CTAs idle
    or run the persistent loop three times, k depths that wrap the operand ring mid-tile, narrow, ragged and
    multi-tile widths, the skip-column append and zero padding of the next layer's tiles, off-boundary output windows;
  * invariants that need no tolerance: row independence, m_dev, determinism;
  * sr_tc_wgrad at its split and accumulator-flush edges, sr_tc_colsum at ragged row counts;
  * negative controls: every bar rejects a reference that lacks the term it guards;
  * argument checks; skip layers whose input n + d_in crosses a multiple of 256, layer by layer and end to end;
  * sr_tc_mlp_backward's value-only reverse sweep, bit for bit against the same chain of raw sr_tc_linear launches.

Every bar is norm-wise (max |err| / max |ref|, tests/helpers.norm_err) unless it says otherwise; every measured error is
printed next to its bar.

Memory safety on an older kernel (bisecting): every layer-level launch here reads and writes only memory the test
allocated, also on a kernel that indexes a reverse launch's stash with pad256 of the launch's own width instead of the
previous layer's (the reverse stashes sit at the front of buffers of that larger size).  The end-to-end case
`skip_k295_ch4` does not: TcMlpFunction allocates each stash at its exact size, so such a kernel reads past it."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NONE, SP, RELU, TANH = 0, 1, 2, 3
ACT = {NONE: "none", SP: "softplus100", RELU: "relu", TANH: "tanh"}
BAR = 1e-5                          # fp32-class GEMM through split-bf16 products (test_gpu_parity's bar)
# act' = sigmoid(100 z) moves by up to 25 dz (tanh' by less): a stash carries 25x the pre-activation error
STASH_FACTOR = 25.0
SENT = 0xA5                         # sentinel byte of every output buffer
INV_SQRT2 = 0.7071067811865476
BM = 128


def _lib():
    from selfreconcode_b200 import _lib as L
    return L.load()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _pad(n, a):
    return (n + a - 1) // a * a


def nerr(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def split2(x):
    """The value the kernels' first two bf16 planes hold for an fp32 x (hi = rn(x), lo = rn(x - hi)), summed in fp32
    as sr_tc_unpack_rows sums them."""
    x = x.float()
    hi = x.bfloat16().float()
    return hi + (x - hi).bfloat16().float()


def bits(t):
    return t.contiguous().view(torch.uint8)


def sentinel(nbytes, dev):
    return torch.full((int(nbytes),), SENT, dtype=torch.uint8, device=dev)


def sentinel_f32(rows, cols, dev):
    return sentinel(rows * cols * 4, dev).view(torch.float32).view(rows, cols)


def poison(nbytes, dev):
    """Scratch that a kernel must write before it is summed: all-ones bytes are NaN as fp32, and a NaN poisons every
    sum that reads an element the kernel left alone."""
    return torch.full((int(nbytes),), 0xFF, dtype=torch.uint8, device=dev)


def pack_rows(lib, x):
    M, K = x.shape
    buf = torch.empty((lib.sr_tc_act_bytes(M, K),), dtype=torch.uint8, device=x.device)
    assert lib.sr_tc_pack_rows(_p(x), M, K, K, _p(buf), None, _stream()) == 0
    return buf


def pack_weights(lib, w):
    N, K = w.shape
    buf = torch.empty((lib.sr_tc_weight_bytes(N, K),), dtype=torch.uint8, device=w.device)
    assert lib.sr_tc_pack_weights(_p(w), N, K, K, _p(buf), _stream()) == 0
    return buf


def unpack(lib, T, M, K, Kpad=None):
    out = torch.empty((M, K), dtype=torch.float32, device=T.device)
    assert lib.sr_tc_unpack_rows(_p(T), M, K, Kpad or _pad(K, 32), _p(out), K, _stream()) == 0
    return out


def linear(lib, A, W, bias, M, N, K, n, act, ch, A_next=None, K_next=0, scale=1.0, skip=None, skip_n=0, out=None,
           out_col0=0, out_n=0, dstash=None, mul_tiles=None, mul_K=0, mul_act=0, mul_scale=1.0, m_dev=None):
    return lib.sr_tc_linear(_p(A), _p(W), _p(bias), M, N, K, n, act, ch, _p(A_next), K_next, scale, _p(skip), skip_n,
                            skip.shape[1] if skip is not None else 0, _p(out), out.shape[1] if out is not None else 0,
                            out_col0, out_n, _p(dstash), _p(mul_tiles), mul_K, mul_act, mul_scale, _p(m_dev), _stream())


# ---------------------------------------------------------------------------------------------------------------------
# fp64 restatement of one sr_tc_linear launch (include/selfrecon_b200.h, LayerArgs in csrc/tc_gemm.cu)
# ---------------------------------------------------------------------------------------------------------------------
def _rows(M, ch, dev):
    """Rows padded to whole points (the kernel's tiles hold zeros past M), value-row index and value-row mask."""
    Mp = _pad(M, ch)
    r = torch.arange(Mp, device=dev)
    return Mp, (r // ch) * ch, (r % ch) == 0


def _zpad(x, Mp):
    return torch.nn.functional.pad(x.double(), (0, 0, 0, Mp - x.shape[0]))


def ref_forward(x, W, b, act, ch, scale, d_prod, relu_mask, use_bias=True):
    """scale * layer(x) [M, N] and the value rows' pre-activation z.  Value rows: act(x W^T + b); tangent rows (ch = 4):
    act'(z of the point's value row) * x W^T, no bias.  The decisions that are ill-conditioned in z come from the
    product's own stored data: the ReLU pattern (`relu_mask`, value rows) and softplus' act' (`d_prod`, the stash)."""
    M = x.shape[0]
    Mp, vrow, isv = _rows(M, ch, x.device)
    acc = _zpad(x, Mp) @ W.double().t()
    z = acc + (b.double() if use_bias else 0.0)
    if act == SP:
        yv = torch.nn.functional.softplus(z, beta=100)
        dt = _zpad(d_prod, Mp)[vrow]
    elif act == RELU:
        m = _zpad(relu_mask, Mp)
        yv = z * m
        dt = m[vrow]
    elif act == TANH:
        yv = torch.tanh(z)
        dt = 1 - torch.tanh(z[vrow]) ** 2
    else:
        yv, dt = z, torch.ones_like(z)
    y = torch.where(isv[:, None], yv, dt * acc)
    return (scale * y)[:M], z[:M]


def ref_reverse(x, Wb, n, mul_act, ch, scale, a_prev, mul_scale, stash, cross=True):
    """Reverse launch: acc = x Wb^T; columns < n: acc * act'(z_prev), columns >= n pass through; all times scale.  act'
    comes from the previous layer's stored activation a_prev (divided by mul_scale) or, when given, from its fp32 stash.
    ch = 4 softplus value rows add 100 (1 - act') sum_c tbar_c t_c over the point's tangent rows."""
    M = x.shape[0]
    Mp, vrow, isv = _rows(M, ch, x.device)
    acc = _zpad(x, Mp) @ Wb.double().t()
    a = _zpad(a_prev, Mp)[:, :n]
    if mul_act == SP:
        d = _zpad(stash[:, :n], Mp)[vrow] if stash is not None else 1 - torch.exp(-100.0 * a[vrow] / mul_scale)
    elif mul_act == RELU:
        d = (a[vrow] > 0).double()
    else:
        d = torch.ones_like(a)
    y = acc.clone()
    y[:, :n] = acc[:, :n] * d
    if ch == 4 and mul_act == SP and cross:
        prod = torch.where(isv[:, None], 0.0, acc[:, :n] * a / mul_scale).view(-1, 4, n).sum(1)
        y[isv, :n] += 100.0 * (1 - d[isv]) * prod
    return (scale * y)[:M]


# ---------------------------------------------------------------------------------------------------------------------
# instantiation x geometry matrix, invariants, negative controls
# ---------------------------------------------------------------------------------------------------------------------
INSTANTIATIONS = ([(act, ch, False) for ch in (1, 4) for act in (NONE, SP, RELU, TANH)] +
                  [(act, ch, True) for ch in (1, 4) for act in (NONE, SP, RELU)])

# M (ch 1, ch 4); K = GEMM depth; N = GEMM width, n = valid columns; A_next with K_next columns, skip_n columns of
# skip_src appended after n, the rest zero; out window [out_col0, out_col0 + out_n); rstash: a reverse launch reads an
# act' stash.  Forward launches always write the stash (its softplus act' is the one the tangent rows used).
GEOMS = {
    # one point on a multi-tile width (a norm-wise bar over a handful of elements would measure their cancellation)
    "M1_K39_N257_skip": dict(M=(1, 4), K=39, N=257, n=257, K_next=320, skip_n=20, scale=INV_SQRT2, out=(0, 257),
                             rstash=False),
    "M127_K32_N3": dict(M=(127, 127), K=32, N=3, n=3, K_next=64, skip_n=0, scale=1.0, out=(0, 3), rstash=True),
    "M128_K192_N473_skip": dict(M=(128, 128), K=192, N=473, n=473, K_next=512, skip_n=39, scale=INV_SQRT2,
                                out=(0, 473), rstash=True),
    "M129_K544_N1": dict(M=(129, 129), K=544, N=1, n=1, K_next=64, skip_n=0, scale=1.0, out=(0, 1), rstash=False),
    # a skip layer's width: N = 256 forward (next input 256 + 39 = 295 columns, past the last column tile);
    # reverse N = 295 over n = 256 (the stash it reads is 256 wide, its own width pads to 512)
    "M300_K64_cross256": dict(M=(300, 300), K=64, N=256, n=256, K_next=320, skip_n=39, scale=INV_SQRT2,
                              out=(0, 256), rstash=True, rev=dict(N=295, K_next=256, skip_n=0, out=(256, 39))),
    # 266 row tiles on 132 CTAs: CTAs 0-1 own three, the others two; K = 544: KC = 17 with NT = 2 wraps the 3-stage
    # ring mid-tile; n < N as in a skip layer's reverse sweep; the window starts off a 32-column boundary
    "big_K544_N512_n473": dict(M=(33923, 33924), K=544, N=512, n=473, K_next=544, skip_n=39, scale=INV_SQRT2,
                               out=(473, 39), rstash=True),
}
BIG = "big_K544_N512_n473"


def _geom(name, mul):
    g = dict(GEOMS[name])
    if mul and "rev" in g:
        g.update(g["rev"])
    return g


def _inputs(dev, g, act, ch, mul, seed):
    """Seeded inputs of one launch (fp32 on the device).  z has std ~0.1, so 100 z spans softplus' curved part."""
    gen = torch.Generator().manual_seed(seed)
    M = g["M"][1 if ch == 4 else 0]
    K, N, n = g["K"], g["N"], g["n"]
    d = dict(M=M)
    d["x"] = torch.randn(M, K, generator=gen).to(dev)
    d["W"] = (torch.randn(N, K, generator=gen) * (0.1 / K ** 0.5)).to(dev)
    d["b"] = (0.05 * torch.randn(N, generator=gen)).to(dev)
    d["skip"] = torch.randn(M, 64, generator=gen).to(dev) if g["skip_n"] else None
    if mul:
        ms = g["scale"]
        kp = _pad(N, 32)
        t = 0.3 * torch.randn(M, kp, generator=gen)
        v = torch.randn(M, kp, generator=gen)
        v = 0.02 * v.abs() if act == SP else (torch.relu(v) if act == RELU else v)
        isv = (torch.arange(M) % ch) == 0
        d["a_prev"] = (ms * torch.where(isv[:, None], v, t)).to(dev)
        d["stash"] = d["stash_buf"] = None
        if g["rstash"] and act == SP:
            # the previous layer's stash, [M][pad256(n)], at the front of a zero-filled buffer as large as
            # [M][pad256(N)]: a kernel that indexed it with this launch's own width reads valid memory, only wrong values
            buf = torch.zeros(M * _pad(max(n, N), 256), device=dev)
            d["stash"] = buf[:M * _pad(n, 256)].view(M, _pad(n, 256))
            d["stash"].copy_(torch.rand(M, _pad(n, 256), generator=gen))
            d["stash_buf"] = buf
    return d


class _Launch:
    """One sr_tc_linear launch of a geometry on fixed inputs; every call writes into fresh sentinel-filled buffers."""

    def __init__(self, lib, dev, g, act, ch, mul, d):
        self.lib, self.dev, self.g, self.act, self.ch, self.mul, self.d = lib, dev, g, act, ch, mul, d
        self.A = pack_rows(lib, d["x"])
        self.Wt = pack_weights(lib, d["W"])
        self.bias = torch.zeros(_pad(g["N"], 256), device=dev)
        if not mul:
            self.bias[:g["N"]] = d["b"]
        self.mt = pack_rows(lib, d["a_prev"]) if mul else None

    def run(self, M=None, m_dev=None):
        g, lib, dev = self.g, self.lib, self.dev
        M = M or self.d["M"]
        o = dict(A_next=sentinel(self.lib.sr_tc_act_bytes(M, g["K_next"]), dev),
                 out=sentinel_f32(M, g["out"][1], dev))
        if self.mul:
            o["stash"] = None
            stash_in = self.d["stash_buf"]
        else:
            o["stash"] = sentinel_f32(M, _pad(g["N"], 256), dev)
            stash_in = o["stash"]
        md = torch.tensor([m_dev], dtype=torch.int32, device=dev) if m_dev is not None else None
        rc = linear(lib, self.A, self.Wt, self.bias, M, g["N"], g["K"], g["n"], NONE if self.mul else self.act, self.ch,
                    A_next=o["A_next"], K_next=g["K_next"], scale=g["scale"], skip=self.d["skip"], skip_n=g["skip_n"],
                    out=o["out"], out_col0=g["out"][0], out_n=g["out"][1], dstash=stash_in,
                    mul_tiles=self.mt, mul_K=_pad(g["N"], 32) if self.mul else 0,
                    mul_act=self.act if self.mul else 0, mul_scale=g["scale"] if self.mul else 1.0, m_dev=md)
        assert rc == 0
        torch.cuda.synchronize()
        return o


def _check_layer(lib, L, o, tag, controls):
    """Every output of a launch against the fp64 contract; the negative controls when `controls`."""
    g, d, act, ch, mul = L.g, L.d, L.act, L.ch, L.mul
    M, N, n = d["M"], g["N"], g["n"]
    c0, cn = g["out"]
    Kn = g["K_next"]
    nxt = unpack(lib, o["A_next"], M, Kn, Kn)
    res = {}
    if mul:
        a_prev = unpack(lib, L.mt, M, N)                         # what the kernel reads: the stored 2-plane value
        ref = ref_reverse(d["x"], d["W"], n, act, ch, g["scale"], a_prev, g["scale"], d["stash"])
    else:
        Mp, vrow, isv = _rows(M, ch, L.dev)
        isv = isv[:M]
        # the product's own ReLU pattern: the stored value-row signs (out window and next-layer tiles)
        mask = torch.zeros(M, N, device=L.dev, dtype=torch.float64)
        mask[:, c0:c0 + cn] = (o["out"] > 0).double()
        mask[:, :n] = (nxt[:, :n] > 0).double()
        ref, z = ref_forward(d["x"], d["W"], d["b"], act, ch, g["scale"], o["stash"][:, :N], mask)
        # the stash: act'(z) of value rows
        st, zv = o["stash"][isv, :N].double(), z[isv]
        zbar = BAR * zv.abs().max().item()                     # the absolute pre-activation error the bar allows
        if act == RELU:
            # only decisions inside the rounding band may come from the product: everywhere else they are fp64's
            firm = zv.abs() > zbar
            assert torch.equal(mask[isv][firm], (zv[firm] > 0).double()), (tag, "ReLU pattern outside the band")
            print("%s: %d of %d value-row ReLU decisions inside the band" % (tag, (~firm).sum().item(), zv.numel()))
        if act in (SP, TANH):
            dref = torch.sigmoid(100 * zv) if act == SP else 1 - torch.tanh(zv) ** 2
            res["stash_abs"] = ((st - dref).abs().max().item(), STASH_FACTOR * zbar)
        else:
            exp = mask[isv] if act == RELU else torch.ones_like(st)
            assert torch.equal(st, exp), (tag, "stash")
    res["out"] = (nerr(o["out"], ref[:, c0:c0 + cn]), BAR)
    # the next layer's tiles store split2 of the fp32 result: up to 2^-18 relative on top of the GEMM's error
    res["next_live"] = (nerr(nxt[:, :n], ref[:, :n]), BAR + 2.0 ** -18)
    # exact: the next layer's tiles hold the split-bf16 value of what `out` received, skip columns and zeros
    if c0 == 0 and cn >= n:
        assert torch.equal(nxt[:, :n], split2(o["out"][:, :n])), (tag, "A_next != split(out)")
    sk = g["skip_n"]
    if sk:
        exp = split2(d["skip"][:, :sk] * torch.tensor(g["scale"], dtype=torch.float32, device=L.dev))
        assert torch.equal(nxt[:, n:n + sk], exp), (tag, "skip columns")
    assert (nxt[:, n + sk:] == 0).all() and not torch.signbit(nxt[:, n + sk:]).any(), (tag, "zero padding")
    if controls and not mul:
        Mp = _pad(M, ch)
        nb, _ = ref_forward(d["x"], d["W"], d["b"], act, ch, g["scale"], o["stash"][:, :N], mask, use_bias=False)
        x1, W1 = d["x"].bfloat16().float(), d["W"].bfloat16().float()
        sp, _ = ref_forward(x1, W1, d["b"], act, ch, g["scale"], o["stash"][:, :N], mask)
        res["ctl_no_bias"] = (nerr(o["out"], nb[:, c0:c0 + cn]), BAR)
        res["ctl_1plane"] = (nerr(o["out"], sp[:, c0:c0 + cn]), BAR)
    if controls and mul and act == SP and ch == 4:
        nc = ref_reverse(d["x"], d["W"], n, act, ch, g["scale"], unpack(lib, L.mt, M, N), g["scale"], d["stash"],
                         cross=False)
        res["ctl_no_cross"] = (nerr(o["out"], nc[:, c0:c0 + cn]), BAR)
    print("%s: %s" % (tag, "  ".join("%s %.2e (bar %.0e)" % (k, v, b) for k, (v, b) in res.items())))
    for k, (v, b) in res.items():
        if k.startswith("ctl_"):
            assert v > b, (tag, k, "the bar must reject this reference", v)
        else:
            assert v < b, (tag, k, v, b)


def _check_invariants(lib, L, full, tag):
    """On the persistent launch: row independence, m_dev, determinism -- bit for bit."""
    g, M, dev = L.g, L.d["M"], L.dev
    Kn = g["K_next"]
    tile_bytes = lib.sr_tc_act_bytes(BM, Kn)
    # determinism
    again = L.run()
    for k, v in full.items():
        if v is not None:
            assert torch.equal(bits(v), bits(again[k])), (tag, "determinism", k)
    # row independence: which CTA owns a tile, and how many tiles it runs, does not change a row's result
    m = 1000
    small = L.run(M=m)
    assert torch.equal(bits(small["out"]), bits(full["out"][:m])), (tag, "row independence: out")
    if small["stash"] is not None:
        assert torch.equal(bits(small["stash"]), bits(full["stash"][:m])), (tag, "row independence: stash")
    assert torch.equal(bits(unpack(lib, small["A_next"], m, Kn, Kn)), bits(unpack(lib, full["A_next"], m, Kn, Kn))), \
        (tag, "row independence: A_next")
    # m_dev < M: rows < m as in the full launch, nothing written past them
    m = 777 if L.ch == 1 else 776
    part = L.run(m_dev=m)
    assert torch.equal(bits(part["out"][:m]), bits(full["out"][:m])), (tag, "m_dev: out rows < m")
    assert (bits(part["out"][m:]) == SENT).all(), (tag, "m_dev: out rows >= m")
    if part["stash"] is not None:
        assert torch.equal(bits(part["stash"][:m]), bits(full["stash"][:m])), (tag, "m_dev: stash rows < m")
        assert (bits(part["stash"][m:]) == SENT).all(), (tag, "m_dev: stash rows >= m")
    assert torch.equal(bits(unpack(lib, part["A_next"], m, Kn, Kn)), bits(unpack(lib, full["A_next"], m, Kn, Kn))), \
        (tag, "m_dev: A_next rows < m")
    assert (part["A_next"][_pad(m, BM) // BM * tile_bytes:] == SENT).all(), (tag, "m_dev: A_next tiles past m")
    # m_dev = 0 writes nothing; m_dev > M behaves as M
    zero = L.run(m_dev=0)
    for k, v in zero.items():
        if v is not None:
            assert (bits(v) == SENT).all(), (tag, "m_dev = 0", k)
    over = L.run(m_dev=M + 1000)
    for k, v in over.items():
        if v is not None:
            assert torch.equal(bits(v), bits(full[k])), (tag, "m_dev > M", k)


@pytest.mark.parametrize("act,ch,mul", INSTANTIATIONS,
                         ids=["%s-%s-ch%d" % ("rev" if m else "fwd", ACT[a], c) for a, c, m in INSTANTIATIONS])
def test_tc_linear_instantiation_matches_fp64(cuda_dev, act, ch, mul):
    lib = _lib()
    for gi, name in enumerate(GEOMS):
        g = _geom(name, mul)
        d = _inputs(cuda_dev, g, act, ch, mul, seed=100 * gi + 10 * act + ch + (5 if mul else 0))
        L = _Launch(lib, cuda_dev, g, act, ch, mul, d)
        full = L.run()
        tag = "%s-%s-ch%d %s" % ("rev" if mul else "fwd", ACT[act], ch, name)
        _check_layer(lib, L, full, tag, controls=name == "M128_K192_N473_skip")
        if name == BIG:
            _check_invariants(lib, L, full, tag)


# ---------------------------------------------------------------------------------------------------------------------
# the reverse launch's act' stash pitch (skip layer input wider than a multiple of 256)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ch", [1, 4])
def test_reverse_stash_pitch_of_wide_skip_layer(cuda_dev, ch):
    """Reverse launch of a skip layer with k = 256 + 39 = 295 inputs over n = 256 continuing columns: the stash it reads
    is the previous layer's, [M][pad256(256) = 256].  The buffer is allocated (zero-filled) at the pitch of this launch's
    own width, pad256(295) = 512 (_inputs), so that a kernel indexing it that way reads valid memory and only gets
    wrong values."""
    lib = _lib()
    g = dict(M=(2400, 2400), K=256, N=295, n=256, K_next=256, skip_n=0, scale=INV_SQRT2, out=(256, 39), rstash=True)
    d = _inputs(cuda_dev, g, SP, ch, True, seed=41)
    M = d["M"]
    assert d["stash_buf"].numel() == M * 512
    L = _Launch(lib, cuda_dev, g, SP, ch, True, d)
    o = L.run()
    a_prev = unpack(lib, L.mt, M, 295)
    ref = ref_reverse(d["x"], d["W"], 256, SP, ch, INV_SQRT2, a_prev, INV_SQRT2, d["stash"])
    e_live = nerr(unpack(lib, o["A_next"], M, 256, 256), ref[:, :256])
    e_skip = nerr(o["out"], ref[:, 256:295])
    print("reverse stash pitch ch=%d: live columns %.2e, skip columns %.2e (bar %.0e)" % (ch, e_live, e_skip, BAR))
    assert e_live < BAR and e_skip < BAR


# ---------------------------------------------------------------------------------------------------------------------
# weight gradient and column sums
# ---------------------------------------------------------------------------------------------------------------------
def _wgrad_split_shape(lib, M, Kd, Kx):
    s = C.c_int(0)
    lib.sr_tc_wgrad_partial_bytes(M, Kd, Kx, C.byref(s))
    halves = 2 * ((M + BM - 1) // BM)
    per = (halves + s.value - 1) // s.value
    runs = [(max(0, min(halves, h0 + per) - h0) + 15) // 16 for h0 in range(0, s.value * per, per)]
    return s.value, per, runs


@pytest.mark.parametrize("M,n,k", [(40000, 512, 512), (640, 512, 1280), (1, 3, 39), (64, 473, 192), (65, 512, 544)])
def test_wgrad_edges_match_fp64(cuda_dev, M, n, k):
    lib = _lib()
    Kd, Kx = _pad(n, 32), _pad(k, 32)
    splits, per, runs = _wgrad_split_shape(lib, M, Kd, Kx)
    if M == 40000:
        assert splits == 16 and per == 40 and max(runs) == 3, "three accumulator runs per split"
    if M == 640:
        assert splits == 6 and runs[-1] == 0, "the last split owns no rows"
    gen = torch.Generator().manual_seed(M + n + k)
    dl = torch.zeros(M, Kd)
    dl[:, :n] = torch.randn(M, n, generator=gen)
    x = torch.zeros(M, Kx)
    x[:, :k] = torch.randn(M, k, generator=gen)
    dl, x = dl.to(cuda_dev), x.to(cuda_dev)
    D, X = pack_rows(lib, dl), pack_rows(lib, x)
    outs = []
    for _ in range(2):
        # the split partials: a split without rows must zero its tile, the first accumulator run must not read it
        part = poison(lib.sr_tc_wgrad_partial_bytes(M, Kd, Kx, None), cuda_dev)
        dW = sentinel_f32(n, k, cuda_dev)
        assert lib.sr_tc_wgrad(_p(D), Kd, _p(X), Kx, M, _p(part), _p(dW), n, k, k, _stream()) == 0
        torch.cuda.synchronize()
        outs.append(dW)
    ref = dl[:, :n].double().t() @ x[:, :k].double()
    assert torch.isfinite(outs[0]).all(), "dW summed a partial entry the kernel never wrote"
    e = nerr(outs[0], ref)
    print("wgrad M=%d n=%d k=%d (%d splits x %d half-tiles, runs %s): %.2e (bar %.0e)"
          % (M, n, k, splits, per, sorted(set(runs)), e, BAR))
    assert e < BAR
    assert torch.equal(bits(outs[0]), bits(outs[1])), "deterministic"


@pytest.mark.parametrize("ch,M", [(1, 1001), (4, 4 * 777), (1, 33923), (4, 33924)])
def test_colsum_matches_fp64(cuda_dev, ch, M):
    lib = _lib()
    K, slices = 39, 64
    x = torch.randn(M, K, generator=torch.Generator().manual_seed(M)).to(cuda_dev)
    T = pack_rows(lib, x)
    part = poison(slices * _pad(K, 32) * 4, cuda_dev).view(torch.float32).view(slices, -1)   # empty slices write 0
    assert lib.sr_tc_colsum(_p(T), M, K, ch, _p(part), slices, _stream()) == 0
    assert torch.isfinite(part).all(), "every slice writes its partial sums"
    got = part.sum(0)[:K]
    vals = unpack(lib, T, M, K).double()
    ref = vals[::ch].sum(0)
    e, e_all = nerr(got, ref), nerr(got, vals.sum(0))
    print("colsum ch=%d M=%d: %.2e (bar %.0e)%s" % (ch, M, e, BAR, "; against all rows (must fail) %.2e" % e_all
                                                     if ch == 4 else ""))
    assert e < BAR
    if ch == 4:
        assert e_all > BAR


# ---------------------------------------------------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------------------------------------------------
def test_tc_linear_rejects_invalid_arguments(cuda_dev):
    """Real, correctly sized buffers: a check that unexpectedly passed would launch on valid memory."""
    from selfreconcode_b200._lib import SR_EINVAL
    lib = _lib()
    M, N, K = 256, 256, 64
    gen = torch.Generator().manual_seed(9)
    A = pack_rows(lib, torch.randn(M, K, generator=gen).to(cuda_dev))
    W = pack_weights(lib, torch.randn(N, K, generator=gen).to(cuda_dev))
    bias = torch.zeros(256, device=cuda_dev)
    mt = pack_rows(lib, torch.randn(M, N, generator=gen).to(cuda_dev))
    out = torch.empty(M, N, device=cuda_dev)
    nxt = torch.empty(lib.sr_tc_act_bytes(M, N), dtype=torch.uint8, device=cuda_dev)
    base = dict(A_next=nxt, K_next=N, out=out, out_n=N)
    bad = {"ch=2": dict(base, ch=2),
           "mul_act=tanh": dict(base, mul_tiles=mt, mul_K=N, mul_act=TANH),
           "mul_K<n_valid": dict(base, mul_tiles=mt, mul_K=N - 32, mul_act=SP),
           "no outputs": dict(ch=1)}
    for name, kw in bad.items():
        kw = dict(kw)
        ch = kw.pop("ch", 1)
        rc = linear(lib, A, W, bias, M, N, K, N, NONE, ch, **kw)
        assert rc == SR_EINVAL, (name, rc)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# sr_tc_mlp_backward's value-only reverse sweep (the tracer's and shading's) against the same chain as raw launches
# ---------------------------------------------------------------------------------------------------------------------
F, T_ = False, True
SWEEPS = {
    # the SDF's value-only view: one skip layer (input 473 + 39), a device-side row count inside a row tile
    "sdf_skip_m_dev": dict(dims=[512, 512, 473, 512, 512, 1], acts=[SP] * 5 + [NONE], skips=[F, F, F, T_, F, F],
                           d_in=39, ld=64, P=5000, m_dev=3001, n_keep=39),
    # the translator: the input layer's launch keeps the 39 positional-encoding columns of its 167 inputs
    "translator_head": dict(dims=[256, 256, 256, 256, 3], acts=[RELU] * 4 + [NONE], skips=[F] * 5, d_in=167, ld=192,
                            P=4100, m_dev=None, n_keep=39),
}


def _sweep_net(lib, dev, c, seed):
    """Packs, a sr_tc_layer array and the kept tiles of one ch = 1 forward sweep of a seeded network."""
    from test_gpu_train import _case
    from selfreconcode_b200._lib import TcLayer
    x0, Ws, bs, _ = _case(dev, 1, c["dims"], c["acts"], c["skips"], c["d_in"], c["ld"], c["P"], seed)
    Ls = []
    arr = (TcLayer * len(Ws))()
    for i, (W, b) in enumerate(zip(Ws, bs)):
        n, k = W.shape
        W = W.to(dev)
        bias = torch.zeros(_pad(n, 256), device=dev)
        bias[:n] = b.to(dev)
        Ls.append(dict(W=W, Wp=pack_weights(lib, W), Wb=pack_weights(lib, W.t().contiguous()), bias=bias,
                       zb=torch.zeros(_pad(k, 256), device=dev), n=n, k=k, act=c["acts"][i], skip=c["skips"][i]))
        a = arr[i]
        a.W, a.Wb, a.bias, a.zero_bias = (Ls[i][t].data_ptr() for t in ("Wp", "Wb", "bias", "zb"))
        a.n, a.k, a.act, a.skip = n, k, Ls[i]["act"], int(Ls[i]["skip"])
    M = c["P"]
    x0 = x0.to(dev)
    A_in = torch.empty(lib.sr_tc_act_bytes(M, c["ld"]), dtype=torch.uint8, device=dev)
    acts = [torch.empty(lib.sr_tc_act_bytes(M, _pad(L["k"], 32)), dtype=torch.uint8, device=dev) for L in Ls[1:]]
    acts_c = (C.c_void_p * len(acts))(*[t.data_ptr() for t in acts])
    out = torch.empty(M, Ls[-1]["n"], device=dev)
    assert lib.sr_tc_mlp_forward(arr, len(Ls), _p(x0), M, c["ld"], c["d_in"], 1, _p(A_in), acts_c, None, _p(out), None,
                                 0, _stream()) == 0
    return Ls, arr, acts, acts_c


def _reverse_by_layers(lib, Ls, cot, bufs, acts, M, m_dev, g_out, g_skip, n_keep, head, d_in):
    """The value-only reverse sweep as one sr_tc_linear launch per layer: pack the cotangent's 32 columns, then from the
    last layer down a reverse launch into the other staging buffer (act' from the previous layer's kept tiles, the skip
    scale as scale and mul_scale, a skip layer's input-gradient part into g_skip), and the input layer into g_out."""
    cur, nxt = bufs
    assert lib.sr_tc_pack_rows(_p(cot), M, 32, 32, _p(cur), _p(m_dev), _stream()) == 0
    K = 32
    for l in range(len(Ls) - 1, -1, -1):
        L = Ls[l]
        scale = INV_SQRT2 if L["skip"] else 1.0
        if l > 0:
            n_prev, Kn = Ls[l - 1]["n"], _pad(Ls[l - 1]["n"], 32)
            gk = g_skip if L["skip"] else None
            assert linear(lib, cur, L["Wb"], L["zb"], M, L["k"], K, n_prev, NONE, 1, A_next=nxt, K_next=Kn, scale=scale,
                          out=gk, out_col0=n_prev, out_n=d_in if gk is not None else 0, mul_tiles=acts[l - 1],
                          mul_K=_pad(L["k"], 32), mul_act=Ls[l - 1]["act"], mul_scale=scale, m_dev=m_dev) == 0
            cur, nxt, K = nxt, cur, Kn
        else:
            Wb, N = (head, n_keep) if head is not None else (L["Wb"], L["k"])
            assert linear(lib, cur, Wb, L["zb"], M, N, K, N, NONE, 1, scale=scale, out=g_out, out_n=n_keep,
                          m_dev=m_dev) == 0


@pytest.mark.parametrize("name", list(SWEEPS))
def test_mlp_backward_value_sweep_matches_layer_launches(cuda_dev, name):
    lib, c = _lib(), SWEEPS[name]
    Ls, arr, acts, acts_c = _sweep_net(lib, cuda_dev, c, seed=23)
    M, n_last, n_keep = c["P"], Ls[-1]["n"], c["n_keep"]
    head = pack_weights(lib, Ls[0]["W"].t()[:n_keep].contiguous()) if n_keep < Ls[0]["k"] else None
    cot = torch.zeros(M, 32, device=cuda_dev)          # sr_tc_trace_mid's rows: zero past the net's outputs
    cot[:, :n_last] = torch.randn(M, n_last, generator=torch.Generator().manual_seed(5)).to(cuda_dev)
    m = c["m_dev"]
    md = torch.tensor([m], dtype=torch.int32, device=cuda_dev) if m is not None else None
    widest = max(_pad(L["n"], 32) for L in Ls[:-1])
    res = []
    for chain in (True, False):
        bufs = [sentinel(lib.sr_tc_act_bytes(M, widest), cuda_dev) for _ in range(2)]
        g_out, g_skip = sentinel_f32(M, 64, cuda_dev), sentinel_f32(M, 64, cuda_dev)
        if chain:
            rc = lib.sr_tc_mlp_backward(arr, len(Ls), M, 64, c["d_in"], 1, _p(cot), 32, None, acts_c, None, _p(bufs[0]),
                                        _p(bufs[1]), None, None, 0, None, None, _p(g_out), _p(g_skip), 64, _p(head),
                                        n_keep, 0, _p(md), _stream())
            assert rc == 0
        else:
            _reverse_by_layers(lib, Ls, cot, bufs, acts, M, md, g_out, g_skip, n_keep, head, c["d_in"])
        torch.cuda.synchronize()
        res.append((g_out, g_skip))
    (g1, s1), (g2, s2) = res
    assert torch.equal(bits(g1), bits(g2)) and torch.equal(bits(s1), bits(s2))
    rows = m if m is not None else M
    assert (bits(g1[:rows, :n_keep]) != SENT).any(dim=1).all() and (bits(g1[:, n_keep:]) == SENT).all()
    assert (bits(g1[rows:]) == SENT).all() and (bits(s1[rows:]) == SENT).all(), "rows past m_dev are left alone"
    if any(L["skip"] for L in Ls):
        assert (bits(s1[:rows, :c["d_in"]]) != SENT).any(dim=1).all()
    else:
        assert (bits(s1) == SENT).all()


def test_mlp_backward_rejects_two_skip_layers_and_invalid_arguments(cuda_dev):
    from selfreconcode_b200._lib import SR_EINVAL, SR_EUNSUPPORTED
    lib = _lib()
    c = dict(SWEEPS["sdf_skip_m_dev"], P=1000)
    Ls, arr, acts, acts_c = _sweep_net(lib, cuda_dev, c, seed=24)
    M = c["P"]
    cot = torch.zeros(M, 32, device=cuda_dev)
    md = torch.tensor([500], dtype=torch.int32, device=cuda_dev)
    bufs = [sentinel(lib.sr_tc_act_bytes(M, 512), cuda_dev) for _ in range(2)]
    g_out, g_skip = sentinel_f32(M, 64, cuda_dev), sentinel_f32(M, 64, cuda_dev)

    def call(arr=arr, gout_ld=32, n_keep=39, fold_skip=0, m_dev=None, head=None):
        return lib.sr_tc_mlp_backward(arr, len(Ls), M, 64, 39, 1, _p(cot), gout_ld, None, acts_c, None, _p(bufs[0]),
                                      _p(bufs[1]), None, None, 0, None, None, _p(g_out), _p(g_skip), 64, _p(head),
                                      n_keep, fold_skip, _p(m_dev), _stream())

    two = type(arr)(*arr)                   # a copy of the layer array with a second skip layer (same widths)
    two[1].skip = 1
    assert arr[1].skip == 0
    assert call(arr=two) == SR_EUNSUPPORTED
    bad = {"gout_ld < n_last": dict(gout_ld=0), "n_keep != k without a head": dict(n_keep=32),
           "head wider than k": dict(n_keep=40, head=Ls[0]["Wb"]), "m_dev with fold_skip": dict(fold_skip=1, m_dev=md)}
    for what, kw in bad.items():
        assert call(**kw) == SR_EINVAL, what
    torch.cuda.synchronize()
    for t in bufs + [g_out, g_skip]:
        assert (bits(t) == SENT).all(), "a refused call launches nothing"


# ---------------------------------------------------------------------------------------------------------------------
# end to end through TcMlpFunction
# ---------------------------------------------------------------------------------------------------------------------
CASES = {
    # the skip layer's input is 256 + 39 = 295 columns: past the forward's last column tile, and the reverse launch's
    # width pads to 512 while the stash it reads is 256 wide.  At 2 800 rows the 256 x 256 layer's weight gradient
    # takes more split scratch than the widest (256 x 320) pair
    "skip_k295_ch4": dict(ch=4, dims=[256, 256, 256, 1], acts=[SP, SP, SP, NONE], skips=[F, F, T_, F], d_in=39, ld=64,
                          P=700, wscale=0.01),
    # 4 x 4400 = 17 600 rows > 132 CTAs x 128: every layer and reverse instantiation runs more than one row tile per CTA
    "sdf_ch4_persistent": dict(ch=4, dims=[512, 473, 512, 257], acts=[SP, SP, SP, NONE], skips=[F, F, T_, F], d_in=39,
                               ld=64, P=4400, wscale=0.01),
    "relu_ch1_persistent": dict(ch=1, dims=[512, 512, 3], acts=[RELU, RELU, NONE], skips=[F] * 3, d_in=167, ld=192,
                                P=20000),
}
# test_gpu_train's bars for networks whose softplus stays in its well-conditioned range (wscale) and for ReLU
TOL = (1e-4, 3e-4)


@pytest.mark.parametrize("name", list(CASES))
def test_tc_mlp_function_edges_vs_fp64_autograd(cuda_dev, name):
    from test_gpu_train import _case, _ref_forward
    from selfreconcode_b200 import train_ops
    from selfreconcode_b200.train_ops import MlpConfig, tc_mlp
    c = CASES[name]
    x0, Ws, bs, R = _case(cuda_dev, c["ch"], c["dims"], c["acts"], c["skips"], c["d_in"], c["ld"], c["P"], 11)
    if "wscale" in c:
        Ws = [w * c["wscale"] for w in Ws[:-1]] + [Ws[-1]]
        bs = [b * c["wscale"] for b in bs[:-1]] + [bs[-1]]
    x0g = x0.to(cuda_dev).requires_grad_(True)
    Wg = [w.to(cuda_dev).requires_grad_(True) for w in Ws]
    bg = [b.to(cuda_dev).requires_grad_(True) for b in bs]
    train_ops.DEBUG_LAST = {}
    out_g = tc_mlp(x0g, MlpConfig(c["acts"], c["skips"], c["d_in"], c["ch"]), Wg, bg)
    dbg, train_ops.DEBUG_LAST = train_ops.DEBUG_LAST, None
    masks = None
    if RELU in c["acts"]:
        masks = [(train_ops.unpack_tiles(a, dbg["M"], dbg["widths"][i]).view(-1, c["ch"], dbg["widths"][i])[:, 0] > 0)
                 for i, a in enumerate(dbg["acts"])] + [None]
    x0r = x0.double().to(cuda_dev).requires_grad_(True)
    Wr = [w.double().to(cuda_dev).requires_grad_(True) for w in Ws]
    br = [b.double().to(cuda_dev).requires_grad_(True) for b in bs]
    out_r = _ref_forward(x0r, Wr, br, c["acts"], c["skips"], c["d_in"], c["ch"], masks)
    Rd = R.to(cuda_dev)
    (out_r * Rd.double()).sum().backward()
    errs = {"out": nerr(out_g.detach(), out_r.detach())}
    (out_g * Rd).sum().backward()
    errs["x0"] = nerr(x0g.grad[:, :c["d_in"]], x0r.grad[:, :c["d_in"]])
    for i in range(len(Ws)):
        errs["W%d" % i] = nerr(Wg[i].grad, Wr[i].grad)
        errs["b%d" % i] = nerr(bg[i].grad, br[i].grad)
    print(name, {k: "%.1e" % v for k, v in errs.items()}, "bars", TOL)
    assert errs["out"] < TOL[0], errs
    assert max(v for k, v in errs.items() if k != "out") < TOL[1], errs
    assert (x0g.grad[:, c["d_in"]:] == 0).all()
