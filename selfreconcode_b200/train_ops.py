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
        if sum(self.skips) > 1:
            # sr_tc_mlp_backward stores each skip layer's input-gradient part into one buffer: a second would overwrite it
            raise RuntimeError("TcMlpFunction: at most one skip layer (got %d)" % sum(self.skips))
        self.d_in = int(d_in)          # width of the embedded input that a skip layer re-appends
        self.ch = int(ch)
        # optional: the module's persistent tensor-core packs (ops.TcNet.layers: W, Wb = W^T, padded bias) of the
        # SAME weights that are passed as tensors -- then nothing is packed per call
        self.packs = packs


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


def _layer_array(cfg, Ws, bs, dev):
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
            W = ops.tc_pack_weights(Ws[i])
            Wb = ops.tc_pack_weights(Ws[i].t())          # [k rows, n cols]
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
            layers, keep = _layer_array(cfg, Ws, bs, dev)
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
            ar = _Arena(dev)
            o_d0 = ar.add(lib.sr_tc_act_bytes(M, wmax))[1]
            o_d1 = ar.add(lib.sr_tc_act_bytes(M, wmax))[1]
            # the split count grows as a layer's dW tiles shrink: a narrower pair can need more scratch than the widest
            kxs = [ld] + [_pad(k, 32) for _, k in shapes[1:]]
            o_part = ar.add(max(lib.sr_tc_wgrad_partial_bytes(M, _pad(n, 32), kx, None)
                                for (n, _), kx in zip(shapes, kxs)))[1]
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
            check(lib.sr_tc_mlp_backward(ctx.layers, L, M, ld, cfg.d_in, ch, _p(g), shapes[-1][0],
                                         C.c_void_p(fa.ptr(ctx.o_in)), ctx.acts_c, ctx.stashes_c,
                                         C.c_void_p(ar.ptr(o_d0)), C.c_void_p(ar.ptr(o_d1)),
                                         C.c_void_p(ar.ptr(o_part)), C.c_void_p(ar.ptr(o_cs)), COLSUM_SLICES, dW_c, db_c,
                                         _p(x0_grad), C.c_void_p(ar.ptr(o_gs)) if o_gs is not None else None, gs_ld,
                                         None, shapes[0][1], 1, None, _stream()), "tc_mlp_backward")
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
                check(lib.sr_tc_embed_backward(_p(pts), P, multires, pw, ch, _p(gx), width, None, 0, _p(gp),
                                               _stream()), "tc_embed_backward")
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


import os as _os


def weight_norm_all(lins):
    """Effective weights of a list of weight-normalised torch Linear modules (weight_v / weight_g), in layer order."""
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
