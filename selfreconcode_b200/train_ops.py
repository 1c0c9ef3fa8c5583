"""Training half of the hot path on the tensor-core engine (reference: model/network.py:599-639 losses with
`create_graph=True`, :774-796 parameter VJPs; utils/utils.py:106-120 compute_Jacobian).

The reference obtains grad f and dD/dp by autograd passes THROUGH the networks and then back-propagates a loss
through those passes (double backward).  Here the derivatives w.r.t. the point are carried FORWARD: every point
is four rows of the layer GEMMs -- the value and its three tangents d/dp_x, d/dp_y, d/dp_z -- so f and grad f
(the offset and its Jacobian) are plain outputs of one forward sweep, and every loss built on them needs just ONE
reverse sweep over the same four rows.  That reverse sweep is first order in the rows but second order in the
network (it contains act''), which is exactly what `loss.backward()` over a `create_graph=True` graph computes.

    TcMlpFunction.apply(x0, cfg, W0, b0, W1, b1, ...) -> out
        x0  [M, ld]  fp32 embedded input rows (M = points * ch; ch = 4: value row then three tangent rows; ch = 1)
        W_l [n, k]   effective weights (weight norm already applied by differentiable torch ops outside)
        out [M, n_last]
    forward : pack -> sr_tc_linear per layer (wgmma split-bf16, activations kept as tiles)
    backward: pack cotangents -> per layer  sr_tc_wgrad (dW = delta^T x, MN-major wgmma GEMM over the kept tiles),
              sr_tc_colsum (db), sr_tc_linear reverse launch (delta_{l-1}; ch = 4 epilogue couples the rows)
No cuBLAS, no torch matmul: torch only carries memory, the embedding and the pointwise loss arithmetic.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import SR_ACT_NONE
from . import ops
from .ops import _p, _pad, _stream, check

INV_SQRT2 = 0.7071067811865476


class MlpConfig:
    """Static description of one MLP stack for TcMlpFunction."""

    def __init__(self, acts, skips, d_in, ch, packs=None):
        self.acts = [int(a) for a in acts]
        self.skips = [bool(s) for s in skips]
        self.d_in = int(d_in)          # width of the embedded input that a skip layer re-appends
        self.ch = int(ch)
        # optional: the module's persistent tensor-core packs (ops.TcNet.layers: W, Wb = W^T, padded bias) of the
        # SAME weights that are passed as tensors -- then nothing is packed per call
        self.packs = packs


def _pack_weights(lib, w):
    w = w.contiguous()
    n, k = w.shape
    buf = torch.empty((lib.sr_tc_weight_bytes(n, k),), dtype=torch.uint8, device=w.device)
    check(lib.sr_tc_pack_weights(_p(w), n, k, w.shape[1], _p(buf), _stream()), "tc_pack_weights")
    return buf


class _Workspace:
    """Scratch shared by backward passes on one (device, stream): wgrad partials, column-sum partials."""
    _pool = {}

    @classmethod
    def get(cls, dev, nbytes):
        key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
        buf = cls._pool.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty((int(nbytes),), dtype=torch.uint8, device=dev)
            cls._pool[key] = buf
        return buf


COLSUM_SLICES = 64
DEBUG_LAST = None      # tests: set to a dict to receive the tiles kept by the last forward (acts, shapes)


def _align(n, a=256):
    return (n + a - 1) // a * a


class _Arena:
    """One device allocation carved into aligned pieces (activation tiles, stashes, scratch): a sweep costs one
    torch.empty instead of one per layer."""

    def __init__(self, dev):
        self.dev = dev
        self.sizes = []

    def add(self, nbytes):
        off = sum(self.sizes)
        self.sizes.append(_align(int(nbytes)))
        return len(self.sizes) - 1, off

    def alloc(self):
        self.buf = torch.empty((max(sum(self.sizes), 1),), dtype=torch.uint8, device=self.dev)
        self.base = self.buf.data_ptr()
        return self

    def ptr(self, off):
        return self.base + off


def _layer_array(lib, cfg, Ws, bs, dev):
    """ctypes array of sr_tc_layer (+ the tensors that must stay alive): the module's persistent packs when given,
    else packed here from the weight tensors."""
    L = len(Ws)
    arr = (_lib.TcLayer * L)()
    keep = []
    for i in range(L):
        n, k = Ws[i].shape
        pk = cfg.packs[i] if cfg.packs is not None else None
        if pk is not None and (pk["n"], pk["k"]) == (n, k):
            W, Wb, bias, zb = pk["W"], pk["Wb"], pk["bias"], pk["zero_bias"]
        else:
            W = _pack_weights(lib, Ws[i])
            Wb = _pack_weights(lib, Ws[i].t().contiguous())          # [k rows, n cols]
            bias = torch.zeros((_pad(n, 256),), dtype=torch.float32, device=dev)
            if bs[i] is not None:
                bias[:n] = bs[i].detach().float()
            zb = torch.zeros((_pad(k, 256),), dtype=torch.float32, device=dev)
        keep += [W, Wb, bias, zb]
        a = arr[i]
        a.W, a.Wb, a.bias, a.zero_bias = W.data_ptr(), Wb.data_ptr(), bias.data_ptr(), zb.data_ptr()
        a.n, a.k, a.act, a.skip = n, k, cfg.acts[i], 1 if cfg.skips[i] else 0
    return arr, keep


class TcMlpFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x0, cfg, *wb):
        lib = _lib.load()
        dev = x0.device
        if not x0.is_cuda:
            raise RuntimeError("TcMlpFunction: CUDA tensors required (no CPU path)")
        x0 = x0.detach().contiguous().float()
        M, ld = x0.shape
        L = len(wb) // 2
        Ws = [wb[2 * i].detach().contiguous().float() for i in range(L)]
        bs = [wb[2 * i + 1] for i in range(L)]
        ch = cfg.ch
        with torch.cuda.device(dev):
            layers, keep = _layer_array(lib, cfg, Ws, bs, dev)
            ar = _Arena(dev)
            _, o_in = ar.add(lib.sr_tc_act_bytes(M, ld))
            o_act, o_st = [], []
            for i in range(L - 1):
                o_act.append(ar.add(lib.sr_tc_act_bytes(M, _pad(Ws[i + 1].shape[1], 32)))[1])
                # softplus(beta=100): act'(z) kept in fp32 for the reverse sweep (1 - act' recomputed from the
                # 16-bit-mantissa activation tiles would carry 100 x 2^-17 of relative error into every gradient)
                o_st.append(ar.add(M * _pad(Ws[i].shape[0], 256) * 4)[1] if cfg.acts[i] == _lib.SR_ACT_SOFTPLUS100 else None)
            ar.alloc()
            acts = (C.c_void_p * max(L - 1, 1))(*[ar.ptr(o) for o in o_act])
            stashes = (C.c_void_p * max(L - 1, 1))(*[ar.ptr(o) if o is not None else None for o in o_st])
            out = torch.empty((M, Ws[-1].shape[0]), dtype=torch.float32, device=dev)
            check(lib.sr_tc_mlp_forward(layers, L, _p(x0), M, ld, cfg.d_in, ch, C.c_void_p(ar.ptr(o_in)), acts, stashes,
                                        _p(out), None, 0, _stream()), "tc_mlp_forward")
            ops.LAUNCHES += L      # check() counted one; a sweep is 1 + L launches
        ctx.cfg, ctx.M, ctx.ld, ctx.L = cfg, M, ld, L
        ctx.arena, ctx.o_in, ctx.acts_c, ctx.stashes_c, ctx.o_act = ar, o_in, acts, stashes, o_act
        ctx.layers, ctx.keep, ctx.shapes = layers, keep, [tuple(w.shape) for w in Ws]
        ctx.has_bias = [b is not None for b in bs]
        if DEBUG_LAST is not None:
            views = [ar.buf[o:o + lib.sr_tc_act_bytes(M, _pad(Ws[i + 1].shape[1], 32))] for i, o in enumerate(o_act)]
            DEBUG_LAST.update(acts=views, M=M, widths=[w.shape[0] for w in Ws], kpads=[_pad(w.shape[1], 32) for w in Ws])
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        lib = _lib.load()
        cfg, M, ld, L, shapes = ctx.cfg, ctx.M, ctx.ld, ctx.L, ctx.shapes
        ch = cfg.ch
        dev = gout.device
        need_x0 = ctx.needs_input_grad[0]
        with torch.cuda.device(dev):
            g = gout.detach().contiguous().float()
            wmax = max(_pad(n, 32) for n, _ in shapes)
            kmax = max([_pad(k, 32) for _, k in shapes[1:]] + [ld])
            ar = _Arena(dev)
            o_d0 = ar.add(lib.sr_tc_act_bytes(M, wmax))[1]
            o_d1 = ar.add(lib.sr_tc_act_bytes(M, wmax))[1]
            o_part = ar.add(lib.sr_tc_wgrad_partial_bytes(M, wmax, kmax, None))[1]
            o_cs = ar.add(COLSUM_SLICES * wmax * 4)[1]
            gs_ld = _pad(cfg.d_in, 4)
            o_gs = ar.add(M * gs_ld * 4)[1] if any(cfg.skips) else None
            ar.alloc()
            # gradients: one buffer, handed back as views
            sizes = [n * k for n, k in shapes] + [n for n, _ in shapes]
            flat = torch.empty((sum(sizes),), dtype=torch.float32, device=dev)
            dWs, dbs, o = [], [], 0
            for n, k in shapes:
                dWs.append(flat[o:o + n * k].view(n, k))
                o += n * k
            for n, _ in shapes:
                dbs.append(flat[o:o + n])
                o += n
            want_w = [ctx.needs_input_grad[2 + 2 * l] for l in range(L)]
            want_b = [ctx.has_bias[l] and ctx.needs_input_grad[3 + 2 * l] for l in range(L)]
            dW_c = (C.c_void_p * L)(*[dWs[l].data_ptr() if want_w[l] else None for l in range(L)])
            db_c = (C.c_void_p * L)(*[dbs[l].data_ptr() if want_b[l] else None for l in range(L)])
            x0_grad = torch.empty((M, ld), dtype=torch.float32, device=dev) if need_x0 else None
            fa = ctx.arena
            check(lib.sr_tc_mlp_backward(ctx.layers, L, M, ld, cfg.d_in, ch, _p(g), C.c_void_p(fa.ptr(ctx.o_in)), ctx.acts_c,
                                         ctx.stashes_c, C.c_void_p(ar.ptr(o_d0)), C.c_void_p(ar.ptr(o_d1)),
                                         C.c_void_p(ar.ptr(o_part)), C.c_void_p(ar.ptr(o_cs)), COLSUM_SLICES, dW_c, db_c,
                                         _p(x0_grad), C.c_void_p(ar.ptr(o_gs)) if o_gs is not None else None, gs_ld,
                                         _stream()), "tc_mlp_backward")
            ops.LAUNCHES += 5 * L
        grads = []
        for l in range(L):
            grads += [dWs[l] if want_w[l] else None, dbs[l] if want_b[l] else None]
        ctx.arena = ctx.keep = None
        return (x0_grad, None) + tuple(grads)


def unpack_tiles(tiles, M, K):
    """tiled split-bf16 activations -> fp32 [M, K] (tests / debugging)."""
    lib = _lib.load()
    out = torch.empty((M, K), dtype=torch.float32, device=tiles.device)
    with torch.cuda.device(tiles.device):
        check(lib.sr_tc_unpack_rows(_p(tiles), M, K, _pad(K, 32), _p(out), K, _stream()), "tc_unpack_rows")
    return out


def tc_mlp(x0, cfg, weights, biases):
    flat = []
    for w, b in zip(weights, biases):
        flat += [w, b]
    return TcMlpFunction.apply(x0, cfg, *flat)


# ------------------------------------------------------------------------------------------------
# Embedding with forward tangents (model/Embedder.py:34-55 + utils/utils.py:40-46), differentiable torch ops
# ------------------------------------------------------------------------------------------------
class EmbedRowsFunction(torch.autograd.Function):
    """embed_rows on two kernels (csrc/tc_gemm.cu: embed_kernel / embed_bwd_kernel) instead of ~40 torch launches
    forward and ~80 backward: x0 rows incl. the latent-code columns; d/dp includes the second derivative of the
    encoding that the tangent rows need; d/d(extra) is the slice of the value rows."""

    @staticmethod
    def forward(ctx, p, extra, multires, pe_w, ch, width):
        lib = _lib.load()
        pts = p.detach().contiguous().float()
        P = pts.shape[0]
        E = extra.shape[1] if extra is not None else 0
        out = torch.empty((P * ch, width), dtype=torch.float32, device=pts.device)
        pw = (C.c_float * 16)(*[float(pe_w[i]) if i < multires else 0.0 for i in range(16)])
        ex = extra.detach().contiguous().float() if extra is not None else None
        with torch.cuda.device(pts.device):
            check(lib.sr_tc_embed(_p(pts), P, multires, pw, ch, _p(ex), None, 1 if ex is not None else 0, E, _p(out), width,
                                  None, None, _stream()), "tc_embed")
        ctx.save_for_backward(pts)
        ctx.meta = (multires, [float(pe_w[i]) for i in range(multires)], ch, width, E)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gx):
        (pts,) = ctx.saved_tensors
        multires, pe_w, ch, width, E = ctx.meta
        lib = _lib.load()
        P = pts.shape[0]
        gx = gx.contiguous().float()
        gp = ge = None
        if ctx.needs_input_grad[0]:
            gp = torch.empty((P, 3), dtype=torch.float32, device=pts.device)
            pw = (C.c_float * 16)(*[pe_w[i] if i < multires else 0.0 for i in range(16)])
            with torch.cuda.device(pts.device):
                check(lib.sr_tc_embed_backward(_p(pts), P, multires, pw, ch, _p(gx), width, _p(gp), _stream()),
                      "tc_embed_backward")
        if E and ctx.needs_input_grad[1]:
            pe = 3 + 6 * multires
            ge = gx.view(P, ch, width)[:, 0, pe:pe + E]
        return gp, ge, None, None, None, None


EMBED_KERNELS = True


def embed_rows(p, multires, pe_w, ch, extra=None, ld=None):
    """p [P,3] -> x0 [P*ch, ld]: row 0 of a point = [p, w_k sin(2^k p), w_k cos(2^k p), ..., extra], rows 1..3 =
    d/dp_c of it (zero for `extra`, which does not depend on p).  `extra` [P,E] (latent code, view, ...)."""
    P = p.shape[0]
    if EMBED_KERNELS and p.is_cuda and p.dtype == torch.float32 and multires <= 8:
        E0 = extra.shape[1] if extra is not None else 0
        width0 = ld if ld is not None else _pad(3 + 6 * multires + E0, 32)
        return EmbedRowsFunction.apply(p, extra, multires, list(pe_w), ch, width0)
    freqs = [float(2 ** k) for k in range(multires)]
    vals = [p]
    for k, fr in enumerate(freqs):
        w = float(pe_w[k])
        vals += [w * torch.sin(p * fr), w * torch.cos(p * fr)]
    val = torch.cat(vals, dim=1)                                       # [P, 3+6L]
    pe = val.shape[1]
    E = extra.shape[1] if extra is not None else 0
    width = ld if ld is not None else _pad(pe + E, 32)
    if ch == 1:
        parts = [val] + ([extra] if extra is not None else [])
        row = torch.cat(parts, dim=1)
        return torch.nn.functional.pad(row, (0, width - row.shape[1]))
    eye = torch.eye(3, dtype=p.dtype, device=p.device)
    tans = [eye.unsqueeze(0).expand(P, 3, 3)]                          # d p / d p_c
    for k, fr in enumerate(freqs):
        w = float(pe_w[k]) * fr
        tans += [torch.diag_embed(w * torch.cos(p * fr)), torch.diag_embed(-w * torch.sin(p * fr))]
    tan = torch.cat(tans, dim=2)                                       # [P, 3(c), 3+6L]
    rows = torch.cat([val.unsqueeze(1), tan], dim=1)                   # [P, 4, pe]
    if extra is not None:
        ex = torch.cat([extra.unsqueeze(1), torch.zeros(P, 3, E, dtype=p.dtype, device=p.device)], dim=1)
        rows = torch.cat([rows, ex], dim=2)
    rows = torch.nn.functional.pad(rows, (0, width - rows.shape[2]))
    return rows.reshape(P * 4, width)


def weight_norm_eff(v, g):
    """torch.nn.utils.weight_norm (dim=0): g * v / ||v||_row -- differentiable elementwise ops, no matmul."""
    if g is None:
        return v
    return v * (g.view(-1, 1) / v.norm(dim=1, keepdim=True))


class WeightNormAllFunction(torch.autograd.Function):
    """Effective weights of several weight-normalised layers: ONE launch forward (sr_weight_norm_forward), ONE launch
    backward (sr_weight_norm_backward) instead of ~12 element-wise / reduce launches per layer per direction.
    Inputs v0, g0, v1, g1, ... (weight_v [n,k], weight_g [n,1]); outputs W0, W1, ... (views of one buffer)."""

    @staticmethod
    def forward(ctx, *vg):
        lib = _lib.load()
        L = len(vg) // 2
        vs = [vg[2 * i].detach().contiguous().float() for i in range(L)]
        gs = [vg[2 * i + 1].detach().reshape(-1).contiguous().float() for i in range(L)]
        dev = vs[0].device
        nk = [tuple(v.shape) for v in vs]
        wbuf = torch.empty((sum(n * k for n, k in nk),), dtype=torch.float32, device=dev)
        inv = torch.empty((sum(n for n, _ in nk),), dtype=torch.float32, device=dev)
        arr = (_lib.WnLayer * L)()
        outs, o, r = [], 0, 0
        for i, (n, k) in enumerate(nk):
            w = wbuf[o:o + n * k].view(n, k)
            c = arr[i]
            c.v, c.g, c.w, c.inv_norm = vs[i].data_ptr(), gs[i].data_ptr(), w.data_ptr(), inv[r:r + n].data_ptr()
            c.gw, c.gv, c.gg, c.n, c.k, c.gw_ld = None, None, None, n, k, k
            outs.append(w)
            o += n * k
            r += n
        with torch.cuda.device(dev):
            check(lib.sr_weight_norm_forward(arr, L, torch.cuda.current_stream().cuda_stream), "weight_norm_forward")
        ctx.save_for_backward(inv, *vs, *gs)
        ctx.nk = nk
        ctx.g_shapes = [vg[2 * i + 1].shape for i in range(L)]
        return tuple(outs)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *gws):
        lib = _lib.load()
        saved = ctx.saved_tensors
        inv = saved[0]
        L = len(ctx.nk)
        vs, gs = saved[1:1 + L], saved[1 + L:1 + 2 * L]
        dev = inv.device
        gvbuf = torch.empty((sum(n * k for n, k in ctx.nk),), dtype=torch.float32, device=dev)
        ggbuf = torch.empty((sum(n for n, _ in ctx.nk),), dtype=torch.float32, device=dev)
        arr = (_lib.WnLayer * L)()
        keep, res, o, r = [], [], 0, 0
        for i, (n, k) in enumerate(ctx.nk):
            gw = gws[i]
            if gw is not None and (gw.dtype != torch.float32 or gw.stride(1) != 1):
                gw = gw.float().contiguous()
            keep.append(gw)
            gv, gg = gvbuf[o:o + n * k].view(n, k), ggbuf[r:r + n]
            c = arr[i]
            c.v, c.g, c.w, c.inv_norm = vs[i].data_ptr(), gs[i].data_ptr(), None, inv[r:r + n].data_ptr()
            c.gw = gw.data_ptr() if gw is not None else None
            c.gv, c.gg, c.n, c.k, c.gw_ld = gv.data_ptr(), gg.data_ptr(), n, k, (gw.stride(0) if gw is not None else k)
            res += [gv, gg.view(ctx.g_shapes[i])]
            o += n * k
            r += n
        with torch.cuda.device(dev):
            check(lib.sr_weight_norm_backward(arr, L, torch.cuda.current_stream().cuda_stream), "weight_norm_backward")
        return tuple(res)


import os as _os

# Off by default: parity-tested (tests/test_gpu_train.py) and 360 launches fewer per optimisation step, but the one
# bench run with it on showed a slower optimizer phase that was never bisected (DESIGN.md section 8).
FUSED_WEIGHT_NORM = _os.environ.get("SELFRECON_B200_FUSED_WN", "0") != "0"


def weight_norm_all(lins, fused=None):
    """Effective weights of a list of weight-normalised torch Linear modules (weight_v / weight_g), in layer order.
    CUDA parameters: one fused launch per direction for up to 12 layers; otherwise the element-wise torch form."""
    if lins and (FUSED_WEIGHT_NORM if fused is None else fused) and lins[0].weight_v.is_cuda and len(lins) <= 12:
        vg = []
        for lin in lins:
            vg += [lin.weight_v, lin.weight_g]
        return list(WeightNormAllFunction.apply(*vg))
    return [weight_norm_eff(lin.weight_v, lin.weight_g) for lin in lins]


# Fused training path switch (SELFRECON_B200_TC_TRAIN=0 routes training through the torch-autograd twin of the
# same math, which tests use as an A/B reference on the same GPU).
TC_TRAIN_ENABLED = _os.environ.get("SELFRECON_B200_TC_TRAIN", "1") != "0"


def small_matmul(a, b):
    """[...,i,j] x [...,j,k] for tiny trailing dims (3x3, 4x4 bone transforms) as a broadcast multiply + sum:
    stays on elementwise kernels (a torch.matmul here would be a cuBLAS batched GEMM launch per call)."""
    return (a.unsqueeze(-1) * b.unsqueeze(-3)).sum(-2)


def small_matvec(m, v):
    """[...,i,j] x [...,j] -> [...,i] without a GEMM launch."""
    return (m * v.unsqueeze(-2)).sum(-1)


def small_mattvec(m, v):
    """[...,j,i]^T x [...,j] -> [...,i]."""
    return (m * v.unsqueeze(-1)).sum(-2)
