"""Torch-facing wrappers over the C ABI (include/selfrecon_b200.h).

torch is plumbing here: it owns device memory and the current stream; every computation is a
call into libselfrecon_b200.so.  All functions require CUDA tensors and raise otherwise --
there is no CPU path in the product (the CPU restatement lives in oracle/ and is only used
by tests and bench baselines).
"""
import ctypes as C
import math

import torch

from . import _lib
from ._lib import MlpDesc, LbsParams, TraceParams
from ._lib import check as _check


import os as _os

# Tensor-core engine switch: large batches go to the wgmma split-BF16 layer GEMMs, small ones to the
# fused fp32 FFMA engine (one persistent kernel, lower latency).  SELFRECON_B200_TC=0 disables it.
TC_ENABLED = _os.environ.get("SELFRECON_B200_TC", "1") != "0"
# 2048: below it a tensor-core trace is launch bound and the fp32 engine (one persistent kernel) is the faster choice
TC_MIN_POINTS = int(_os.environ.get("SELFRECON_B200_TC_MIN_POINTS", "2048"))

# Borderline decisions on tensor-core values are re-taken on the fp32 FFMA engine (DESIGN.md section 4):
# TC_EPS_F bounds the engine's absolute error on an SDF value (split-BF16 with fp32 accumulation, csrc/tc_gemm.cu),
# TC_EPS_A (degrees) the error of the ray/point angle that follows from D(p)'s.
TC_EPS_F = float(_os.environ.get("SELFRECON_B200_TC_EPS_F", "4e-5"))
TC_EPS_A = float(_os.environ.get("SELFRECON_B200_TC_EPS_A", "1e-3"))
TC_REFINE = _os.environ.get("SELFRECON_B200_TC_REFINE", "1") != "0"
# The tracer's in-loop fp32 re-test costs one latency-bound FFMA launch per iteration and cannot remove the dominant source of per-ray divergence (sign(f) in the update when |f| is below the
# engine's error, DESIGN.md section 4): off by default, kept for experiments.
TC_REFINE_TRACE = _os.environ.get("SELFRECON_B200_TC_REFINE_TRACE", "0") != "0"
TC_DUAL_STREAM = _os.environ.get("SELFRECON_B200_TC_DUAL_STREAM", "1") != "0"

import itertools as _it
_uid_counter = _it.count()
LAUNCHES = 0  # kernels launched by this module since it was last reset (bench.py reads it)

_KERNELS_PER_CALL = {"mc_count": 3}


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(code, what):
    """C-ABI return code -> RuntimeError; also counts the kernels the call launched."""
    global LAUNCHES
    _check(code, what)
    LAUNCHES += _KERNELS_PER_CALL.get(what, 1)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("selfrecon_b200: expected a CUDA tensor (no CPU fallback)")


# ------------------------------------------------------------------------------------------------
# FastMinv  (FastMinv/M3x3Inv.cpp:12-59)
# ------------------------------------------------------------------------------------------------
def minv3x3(ms):
    _need_cuda(ms)
    n = ms.shape[0]
    invs = torch.empty((n, 3, 3), dtype=ms.dtype, device=ms.device)
    checks = torch.empty((n,), dtype=torch.bool, device=ms.device)
    lib = _lib.load()
    with torch.cuda.device(ms.device):
        fn = lib.sr_minv3x3_f32 if ms.dtype == torch.float32 else lib.sr_minv3x3_f64
        check(fn(_p(ms), _p(invs), _p(checks), n, _stream()), "minv3x3")
    return invs, checks


def minv3x3_backward(grads, invs):
    _need_cuda(grads, invs)
    n = invs.shape[0]
    outs = torch.empty((n, 3, 3), dtype=invs.dtype, device=invs.device)
    lib = _lib.load()
    with torch.cuda.device(invs.device):
        fn = lib.sr_minv3x3_bwd_f32 if invs.dtype == torch.float32 else lib.sr_minv3x3_bwd_f64
        check(fn(_p(grads), _p(invs), _p(outs), n, _stream()), "minv3x3_bwd")
    return outs


def raster_mesh(verts_screen, faces, H, W):
    """verts_screen [N,V,3] (pixel x, pixel y, depth), faces [F,3] int64 -> (pix_to_face [N,H,W,1] int64,
    bary [N,H,W,1,3], zbuf [N,H,W,1]): pytorch3d Fragments layout with one face per pixel."""
    _need_cuda(verts_screen, faces)
    vs = verts_screen.detach().contiguous().float()
    fc = faces.contiguous().to(torch.int64)
    N, V, _ = vs.shape
    F = fc.shape[0]
    dev = vs.device
    keys = torch.empty((N, H, W), dtype=torch.int64, device=dev)
    p2f = torch.empty((N, H, W, 1), dtype=torch.int64, device=dev)
    bary = torch.empty((N, H, W, 1, 3), dtype=torch.float32, device=dev)
    zbuf = torch.empty((N, H, W, 1), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().sr_raster_mesh(_p(vs), _p(fc), N, V, F, int(H), int(W), _p(keys), _p(p2f), _p(bary),
                                         _p(zbuf), _stream()), "raster_mesh")
    return p2f, bary, zbuf


_KERNELS_PER_CALL["raster_mesh"] = 2


def svals3x3(J, want_v=True):
    """J [n,3,3] f32 CUDA -> (singular values [n,3] descending, V [n,3,3] | None)."""
    _need_cuda(J)
    J = J.contiguous().float()
    n = J.shape[0]
    S = torch.empty((n, 3), dtype=torch.float32, device=J.device)
    V = torch.empty((n, 3, 3), dtype=torch.float32, device=J.device) if want_v else None
    with torch.cuda.device(J.device):
        check(_lib.load().sr_svals3x3_f32(_p(J), _p(S), _p(V), n, _stream()), "svals3x3")
    return S, V


def svals3x3_backward(J, S, V, gS):
    _need_cuda(J, S, V, gS)
    n = J.shape[0]
    gJ = torch.empty((n, 3, 3), dtype=torch.float32, device=J.device)
    with torch.cuda.device(J.device):
        check(_lib.load().sr_svals3x3_bwd_f32(_p(J.contiguous()), _p(S.contiguous()), _p(V.contiguous()),
                                              _p(gS.contiguous().float()), _p(gJ), n, _stream()), "svals3x3_bwd")
    return gJ


# ------------------------------------------------------------------------------------------------
# Marching cubes (MCGpu/MCGpu.cpp:20-56)
# ------------------------------------------------------------------------------------------------
_mc_work = {}


def marching_cubes(sdfs, xstep=1.0, ystep=1.0, zstep=1.0, xmin=0.0, ymin=0.0, zmin=0.0, iso=0.0,
                   i_offset=0):
    """sdfs [NX,NY,NZ] f32 contiguous CUDA -> (vertices [V,3] f32, faces [F,3] i64), canonical
    (deterministic) order.  One device->host read of the two counters, like the reference."""
    _need_cuda(sdfs)
    nx, ny, nz = sdfs.shape
    lib = _lib.load()
    dev = sdfs.device
    with torch.cuda.device(dev):
        wb = lib.sr_mc_work_bytes(nx, ny, nz)
        key = (dev.index, torch.cuda.current_stream().cuda_stream)
        work = _mc_work.get(key)
        if work is None or work.numel() < wb:
            work = torch.empty((wb,), dtype=torch.uint8, device=dev)
            _mc_work[key] = work  # grows monotonically, like the reference's per-device scratch
        counts = torch.empty((2,), dtype=torch.int32, device=dev)
        check(lib.sr_mc_count(_p(sdfs), nx, ny, nz, float(iso), _p(work), _p(counts), _stream()),
              "mc_count")
        nv, nf = counts.tolist()  # the one blocking read-back
        verts = torch.empty((nv, 3), dtype=torch.float32, device=dev)
        faces = torch.empty((nf, 3), dtype=torch.int64, device=dev)
        if nv or nf:
            check(lib.sr_mc_emit(_p(sdfs), nx, ny, nz, float(iso), float(xstep), float(ystep),
                                 float(zstep), float(xmin), float(ymin), float(zmin), int(i_offset),
                                 _p(work),
                                 _p(verts), nv, _p(faces), nf, _stream()), "mc_emit")
    return verts, faces


def marching_cubes_count(sdfs, iso=0.0):
    """(number of vertices, number of faces) marching_cubes() would produce: the classification + scan half of
    the sweep only (used by the slab-sharded extraction to split a slab's output into own / halo parts)."""
    _need_cuda(sdfs)
    nx, ny, nz = sdfs.shape
    lib = _lib.load()
    dev = sdfs.device
    with torch.cuda.device(dev):
        wb = lib.sr_mc_work_bytes(nx, ny, nz)
        key = (dev.index, torch.cuda.current_stream().cuda_stream, "count")
        work = _mc_work.get(key)
        if work is None or work.numel() < wb:
            work = torch.empty((wb,), dtype=torch.uint8, device=dev)
            _mc_work[key] = work
        counts = torch.empty((2,), dtype=torch.int32, device=dev)
        check(lib.sr_mc_count(_p(sdfs), nx, ny, nz, float(iso), _p(work), _p(counts), _stream()), "mc_count")
        nv, nf = counts.tolist()
    return nv, nf


# ------------------------------------------------------------------------------------------------
# interp2x_boundary  (MCAcc/cuda/interp2x_boundary3d.cpp:17-36)
# ------------------------------------------------------------------------------------------------
def interp2x3d_forward(inp, balance):
    _need_cuda(inp)
    b, c, d, h, w = inp.shape
    out = torch.empty((b, c, 2 * d - 1, 2 * h - 1, 2 * w - 1), dtype=inp.dtype, device=inp.device)
    bnd = torch.empty(out.shape, dtype=torch.bool, device=inp.device)
    lib = _lib.load()
    with torch.cuda.device(inp.device):
        check(lib.sr_interp2x3d_fwd_f32(_p(inp), _p(out), _p(bnd), b * c, d, h, w, float(balance),
                                        _stream()), "interp2x3d_fwd")
    return out, bnd


def interp2x3d_backward(grad_out):
    _need_cuda(grad_out)
    b, c, od, oh, ow = grad_out.shape
    d, h, w = (od + 1) // 2, (oh + 1) // 2, (ow + 1) // 2
    gin = torch.empty((b, c, d, h, w), dtype=grad_out.dtype, device=grad_out.device)
    lib = _lib.load()
    with torch.cuda.device(grad_out.device):
        check(lib.sr_interp2x3d_bwd_f32(_p(grad_out), _p(gin), b * c, d, h, w, _stream()),
              "interp2x3d_bwd")
    return gin


def interp2x2d_forward(inp, balance):
    _need_cuda(inp)
    b, c, h, w = inp.shape
    out = torch.empty((b, c, 2 * h - 1, 2 * w - 1), dtype=inp.dtype, device=inp.device)
    bnd = torch.empty(out.shape, dtype=torch.bool, device=inp.device)
    lib = _lib.load()
    with torch.cuda.device(inp.device):
        check(lib.sr_interp2x2d_fwd_f32(_p(inp), _p(out), _p(bnd), b * c, h, w, float(balance),
                                        _stream()), "interp2x2d_fwd")
    return out, bnd


def interp2x2d_backward(grad_out):
    _need_cuda(grad_out)
    b, c, oh, ow = grad_out.shape
    h, w = (oh + 1) // 2, (ow + 1) // 2
    gin = torch.empty((b, c, h, w), dtype=grad_out.dtype, device=grad_out.device)
    lib = _lib.load()
    with torch.cuda.device(grad_out.device):
        check(lib.sr_interp2x2d_bwd_f32(_p(grad_out), _p(gin), b * c, h, w, _stream()),
              "interp2x2d_bwd")
    return gin


# ------------------------------------------------------------------------------------------------
# GridSamplerMine  (MCAcc/cuda/GridSamplerMine.cpp:73-96)
# ------------------------------------------------------------------------------------------------
def _istr(t):
    return (C.c_int64 * 5)(*t.stride())


def _gs_suffix(t):
    if t.dtype == torch.float32:
        return "f32"
    if t.dtype == torch.float64:
        return "f64"
    raise RuntimeError("grid_sampler_3d: only float32/float64 are supported")


def grid_sample3d_forward(inp, grid, want_corner_idx=False):
    _need_cuda(inp, grid)
    N, Cc, D, H, W = inp.shape
    Do, Ho, Wo = grid.shape[1:4]
    P = Do * Ho * Wo
    g = grid.reshape(N, P, 3).contiguous()
    out = torch.empty((N, Cc, Do, Ho, Wo), dtype=inp.dtype, device=inp.device)
    cidx = torch.empty((N, P, 3), dtype=torch.int32, device=inp.device) if want_corner_idx else None
    lib = _lib.load()
    with torch.cuda.device(inp.device):
        fn = getattr(lib, "sr_grid_sample3d_fwd_" + _gs_suffix(inp))
        check(fn(_p(inp), _istr(inp), _p(g), _p(out), _p(cidx), N, Cc, D, H, W, P, _stream()),
              "grid_sample3d_fwd")
    return (out, cidx) if want_corner_idx else out


def grid_sample3d_backward(inp, grid, grad_output):
    _need_cuda(inp, grid, grad_output)
    N, Cc, D, H, W = inp.shape
    Do, Ho, Wo = grid.shape[1:4]
    P = Do * Ho * Wo
    g = grid.reshape(N, P, 3).contiguous()
    go = grad_output.reshape(N, Cc, P).contiguous()
    ginp = torch.zeros((N, Cc, D, H, W), dtype=inp.dtype, device=inp.device)
    ggrid = torch.empty((N, P, 3), dtype=inp.dtype, device=inp.device)
    lib = _lib.load()
    with torch.cuda.device(inp.device):
        fn = getattr(lib, "sr_grid_sample3d_bwd_" + _gs_suffix(inp))
        check(fn(_p(inp), _istr(inp), _p(g), _p(go), _p(ginp), _p(ggrid), N, Cc, D, H, W, P,
                 _stream()), "grid_sample3d_bwd")
    return ginp, ggrid.reshape(grid.shape)


def grid_sample3d_dbackward(gg_input, gg_grid, inp, grid, grad_output):
    _need_cuda(gg_input, gg_grid, inp, grid, grad_output)
    N, Cc, D, H, W = inp.shape
    Do, Ho, Wo = grid.shape[1:4]
    P = Do * Ho * Wo
    g = grid.reshape(N, P, 3).contiguous()
    go = grad_output.reshape(N, Cc, P).contiguous()
    ggi = gg_input.contiguous()
    ggg = gg_grid.reshape(N, P, 3).contiguous()
    ginp = torch.zeros((N, Cc, D, H, W), dtype=inp.dtype, device=inp.device)
    ggrid = torch.empty((N, P, 3), dtype=inp.dtype, device=inp.device)
    ggout = torch.empty((N, Cc, P), dtype=inp.dtype, device=inp.device)
    lib = _lib.load()
    with torch.cuda.device(inp.device):
        fn = getattr(lib, "sr_grid_sample3d_dbwd_" + _gs_suffix(inp))
        check(fn(_p(ggi), _p(ggg), _p(inp), _istr(inp), _p(g), _p(go), _p(ginp), _p(ggrid),
                 _p(ggout), N, Cc, D, H, W, P, _stream()), "grid_sample3d_dbwd")
    return ginp, ggrid.reshape(grid.shape), ggout.reshape(grad_output.shape)


# ------------------------------------------------------------------------------------------------
# Fused MLP stacks
# ------------------------------------------------------------------------------------------------
def _pad(x, m):
    return (x + m - 1) // m * m


class FusedMLP:
    """Folded (weight-norm applied, transposed, padded) copy of an MLP's parameters plus the
    sr_mlp_desc that points at it.  `linears` is a list of dicts with keys
    v [n,k], g [n] or None, b [n] or None, act (SR_ACT_*), skip (bool)."""

    def __init__(self, d_in, multires, device):
        self.d_in = int(d_in)
        self.multires = int(multires)
        self.device = torch.device(device)
        self.bufs = []
        self.desc = MlpDesc()
        self._sig = None
        self.uid = next(_uid_counter)   # identity for caches (id() can be recycled)

    def fold(self, linears, pe_w=None):
        """Folds (weight norm applied, transposed, padded) the given layers into this object's device buffers.
        The buffers are allocated on the first call and REUSED afterwards (`refold`): descriptors, tensor-core
        packs and captured CUDA graphs that point at them stay valid when the parameters change."""
        d = self.desc
        d.n_layers = len(linears)
        d.d_in = self.d_in
        d.multires = self.multires
        pw = pe_w if pe_w is not None else [1.0] * self.multires
        for i in range(16):
            d.pe_w[i] = float(pw[i]) if i < len(pw) else 0.0
        if len(linears) > _lib.SR_MLP_MAX_LAYERS:
            raise RuntimeError("FusedMLP: too many layers")
        self._linears = linears
        self._lay = []
        with torch.cuda.device(self.device):
            for i, L in enumerate(linears):
                n, k = L["v"].shape
                _need_cuda(L["v"])
                npad, kpad = _pad(n, 128), _pad(k, 8)
                if npad > 512 or kpad > 512:
                    raise RuntimeError("FusedMLP: layer %dx%d exceeds the 512-wide engine" % (n, k))
                wt = torch.empty((kpad, npad), dtype=torch.float32, device=self.device)
                bias = torch.empty((npad,), dtype=torch.float32, device=self.device)
                wb = torch.empty((_pad(n, 8), _pad(k, 128)), dtype=torch.float32, device=self.device)
                self._lay.append(dict(wt=wt, bias=bias, wb=wb, n=n, k=k, npad=npad, kpad=kpad))
                ly = d.layer[i]
                ly.wt, ly.bias, ly.wb = wt.data_ptr(), bias.data_ptr(), wb.data_ptr()
                ly.k, ly.n, ly.kpad, ly.npad = k, n, kpad, npad
                ly.act = int(L["act"])
                ly.skip = 1 if L.get("skip") else 0
        self.bufs = [t for e in self._lay for t in (e["wt"], e["bias"], e["wb"])]
        self._children = []
        self.version = 0
        self.refold()
        return self

    def refold(self):
        """Re-runs the fold kernels from the current parameter values into the existing buffers, then refreshes
        everything derived from them (truncated views, tensor-core packs)."""
        lib = _lib.load()
        with torch.cuda.device(self.device):
            for e, L in zip(self._lay, self._linears):
                v = L["v"].detach().contiguous().float()
                g, b = L.get("g"), L.get("b")
                g = g.detach().contiguous().float().view(-1) if g is not None else None
                b = b.detach().contiguous().float() if b is not None else None
                check(lib.sr_fold_linear(_p(v), _p(g), _p(b), e["n"], e["k"], e["npad"], e["kpad"], _p(e["wt"]),
                                         _p(e["bias"]), _p(e["wb"]), _stream()), "fold_linear")
        self.version += 1
        for c in self._children:
            c._refresh_from_parent()
        tc = getattr(self, "_tc", None)
        if tc is not None:
            tc.repack()
        return self

    def set_pe_weights(self, pe_w):
        for i in range(16):
            self.desc.pe_w[i] = float(pe_w[i]) if i < len(pe_w) else 0.0

    def truncated_last(self, n_out):
        """A view of the same network whose last layer only produces the first n_out outputs
        (e.g. the SDF value without the 256-d feature): same buffers, narrower npad."""
        t = FusedMLP(self.d_in, self.multires, self.device)
        C.memmove(C.byref(t.desc), C.byref(self.desc), C.sizeof(MlpDesc))
        last = t.desc.layer[t.desc.n_layers - 1]
        e = self._lay[-1]
        npad = _pad(n_out, 128)
        t._own = None
        if npad != e["npad"]:
            # W_T rows are npad-strided, so a narrower view needs its own copy of the columns
            t._own = (e["wt"][:, :npad].contiguous(), e["bias"][:npad].contiguous(), npad)
            last.wt = t._own[0].data_ptr()
            last.bias = t._own[1].data_ptr()
            last.npad = npad
        last.n = n_out
        t._parent = self
        t._lay = self._lay[:-1] + [dict(e, n=n_out, npad=npad, wt=t._own[0] if t._own else e["wt"],
                                        bias=t._own[1] if t._own else e["bias"])]
        t.bufs = [x for x in (t._own[:2] if t._own else [])]
        t._children = []
        t.version = self.version
        self._children.append(t)
        return t

    def _refresh_from_parent(self):
        if self._own is not None:
            e = self._parent._lay[-1]
            self._own[0].copy_(e["wt"][:, :self._own[2]])
            self._own[1].copy_(e["bias"][:self._own[2]])
        self.version = self._parent.version
        tc = getattr(self, "_tc", None)
        if tc is not None:
            tc.repack()


def annealing_weights(multires, ratio):
    """utils/utils.py:40-46 (one weight per band; the reference repeats each twice)."""
    if ratio is None:
        return [1.0] * multires
    if ratio <= 0:
        return [0.0] * multires
    alpha = ratio * multires
    return [(1.0 - math.cos(math.pi * min(max(alpha - float(i), 0.0), 1.0))) / 2.0
            for i in range(multires)]


def sdf_forward(net, pts, want_grad=False, nfeat=0):
    _need_cuda(pts)
    pts = pts.contiguous().float()
    P = pts.shape[0]
    dev = pts.device
    sdf = torch.empty((P,), dtype=torch.float32, device=dev)
    grad = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_grad else None
    feat = torch.empty((P, nfeat), dtype=torch.float32, device=dev) if nfeat else None
    lib = _lib.load()
    with torch.cuda.device(dev):
        check(lib.sr_sdf_forward(C.byref(net.desc), _p(pts), P, _p(sdf), _p(grad), _p(feat),
                                 int(nfeat), _stream()), "sdf_forward")
    return sdf, grad, feat


_band_scratch = {}
SMALL_REFINE = _os.environ.get("SELFRECON_B200_SMALL_REFINE", "1") != "0"
SMALL_CAP = 4096
_KERNELS_PER_CALL["sdf_forward_small"] = 10


def sdf_refine_band(net, pts, sdf, center=0.0, eps=None):
    """In place: every sdf[i] with |sdf[i] - center| < eps is re-evaluated by the fp32 FFMA engine
    (device-side list + count, no host sync).  `net` is the FusedMLP the values came from."""
    _need_cuda(pts, sdf)
    eps = TC_EPS_F if eps is None else float(eps)
    P = sdf.numel()
    if P == 0:
        return sdf
    dev = sdf.device
    lib = _lib.load()
    with torch.cuda.device(dev):
        key = (dev.index, torch.cuda.current_stream().cuda_stream)
        buf = _band_scratch.get(key)
        if buf is None or buf.numel() < P + 1:
            buf = torch.empty((max(P + 1, 1 << 16),), dtype=torch.int32, device=dev)
            _band_scratch[key] = buf
        cnt, lst = buf[0:1], buf[1:]
        cnt.zero_()
        check(lib.sr_band_select(_p(sdf), P, float(center), eps, _p(lst), _p(cnt), _stream()), "band_select")
        if SMALL_REFINE:
            # short lists: one column-split launch per layer instead of the persistent engine's per-tile latency;
            # the list is longer than SMALL_CAP only in degenerate cases -- then the persistent engine takes all of it
            wkey = key + ("small",)
            work = _band_scratch.get(wkey)
            if work is None:
                work = torch.empty((lib.sr_sdf_small_work_bytes(SMALL_CAP),), dtype=torch.uint8, device=dev)
                _band_scratch[wkey] = work
            check(lib.sr_sdf_forward_small(C.byref(net.desc), _p(pts), P, _p(lst), _p(cnt), _p(sdf), _p(work),
                                           SMALL_CAP, _stream()), "sdf_forward_small")
            over = _band_scratch.get(key + ("over",))
            if over is None:
                over = torch.empty((1,), dtype=torch.int32, device=dev)
                _band_scratch[key + ("over",)] = over
            torch.clamp(cnt - SMALL_CAP, min=0, out=over)
            if P > SMALL_CAP:
                check(lib.sr_sdf_forward_indexed(C.byref(net.desc), _p(pts), P, _p(lst[SMALL_CAP:]), _p(over), _p(sdf),
                                                 _stream()), "sdf_forward_indexed")
        else:
            check(lib.sr_sdf_forward_indexed(C.byref(net.desc), _p(pts), P, _p(lst), _p(cnt), _p(sdf), _stream()),
                  "sdf_forward_indexed")
    return sdf


class LbsState:
    """Device-side LBS inputs: channels-last weight volume + per-frame bone transforms."""

    def __init__(self, ws_ncdhw, bmin, bmax, Js, parents, init_pose_inv):
        _need_cuda(ws_ncdhw)
        dev = ws_ncdhw.device
        _, c, D, H, W = ws_ncdhw.shape
        assert c == 24
        self.D, self.H, self.W = D, H, W
        self.device = dev
        self.ws_cl = torch.empty((D, H, W, 24), dtype=torch.float32, device=dev)
        lib = _lib.load()
        with torch.cuda.device(dev):
            check(lib.sr_lbs_weights_to_channels_last(_p(ws_ncdhw.contiguous().float()),
                                                      _p(self.ws_cl), D, H, W, _stream()),
                  "lbs_weights_to_channels_last")
        self.bmin = [float(x) for x in bmin.view(-1).tolist()]
        self.bmax = [float(x) for x in bmax.view(-1).tolist()]
        self.Js = Js.detach().contiguous().float().view(24, 3)
        self.parents = torch.as_tensor(parents, dtype=torch.int32, device=dev).contiguous()
        self.ipi = init_pose_inv.detach().contiguous().float() if init_pose_inv is not None else None
        self.A = None
        self.trans = None
        self.params = LbsParams()

    def set_pose(self, poses, trans, want_posed_joints=False):
        """poses [F,24,3] axis-angle, trans [F,3] -> bone transforms on device."""
        F = poses.shape[0]
        poses = poses.detach().contiguous().float().view(F, 24, 3)
        self.trans = trans.detach().contiguous().float().view(F, 3)
        self.A = torch.empty((F, 24, 4, 4), dtype=torch.float32, device=self.device)
        pj = torch.empty((F, 24, 3), dtype=torch.float32, device=self.device) if want_posed_joints else None
        lib = _lib.load()
        with torch.cuda.device(self.device):
            check(lib.sr_lbs_bone_transforms(_p(poses), _p(self.Js), _p(self.parents), _p(self.ipi),
                                             F, _p(self.A), _p(pj), _stream()), "lbs_bone_transforms")
        p = self.params
        p.ws_cl = self.ws_cl.data_ptr()
        p.D, p.H, p.W = self.D, self.H, self.W
        for i in range(3):
            p.bmin[i] = self.bmin[i]
            p.bmax[i] = self.bmax[i]
        p.A = self.A.data_ptr()
        p.trans = self.trans.data_ptr()
        p.F = F
        return pj


def _lbs_ref(lbs):
    return C.byref(lbs.params) if lbs is not None else None


def deform_forward(net, lbs, pts, batch_inds, conds, want_jac=False, want_offset=False,
                   want_corner_idx=False, pts_per_frame=0):
    _need_cuda(pts)
    pts = pts.contiguous().float().view(-1, 3)
    P = pts.shape[0]
    dev = pts.device
    conds = conds.detach().contiguous().float() if conds is not None else None
    condlen = conds.shape[-1] if conds is not None else 0
    bi = batch_inds.contiguous().to(torch.int64) if batch_inds is not None else None
    d = torch.empty((P, 3), dtype=torch.float32, device=dev)
    off = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_offset else None
    jac = torch.empty((P, 3, 3), dtype=torch.float32, device=dev) if want_jac else None
    ci = torch.empty((P, 3), dtype=torch.int32, device=dev) if want_corner_idx else None
    lib = _lib.load()
    with torch.cuda.device(dev):
        check(lib.sr_deform_forward(C.byref(net.desc), _lbs_ref(lbs), _p(pts), _p(bi),
                                    int(pts_per_frame), _p(conds), condlen, P, _p(d), _p(off),
                                    _p(jac), _p(ci), _stream()), "deform_forward")
    return d, off, jac, ci


def render_forward(net, pts, normals, views, feat):
    _need_cuda(pts, normals, views)
    P = pts.shape[0]
    dev = pts.device
    nfeat = feat.shape[1] if feat is not None else 0
    rgb = torch.empty((P, 3), dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        check(lib.sr_render_forward(C.byref(net.desc), _p(pts.contiguous().float()),
                                    _p(normals.contiguous().float()), _p(views.contiguous().float()),
                                    _p(feat.contiguous().float() if feat is not None else None),
                                    nfeat, P, _p(rgb), _stream()), "render_forward")
    return rgb


_scratch = {}


_host_cache = {}


def _host_floats(t):
    """Host copy of a small device tensor (camera centre), cached by (storage, version): the blocking
    device->host read happens once per tensor value, not once per trace."""
    if not t.is_cuda:
        return tuple(float(x) for x in t.detach().reshape(-1).tolist())
    key = (t.device.index, t.data_ptr(), t._version, t.numel())
    v = _host_cache.get(key)
    if v is None:
        if len(_host_cache) > 64:
            _host_cache.clear()
        v = tuple(float(x) for x in t.detach().reshape(-1).tolist())
        _host_cache[key] = v
    return v


def _trace_scratch(dev):
    """act'(z) stash of the reverse-mode tracer (one region per SM), one per (device, stream) so that
    traces running concurrently on two streams do not share it."""
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
    if key not in _scratch:
        n = _lib.load().sr_trace_scratch_bytes()
        _scratch[key] = torch.empty((n // 4,), dtype=torch.float32, device=dev)
    return _scratch[key]


def trace_surface_points(sdf_net, def_net, lbs, cam_pos, rays, init_pts, batch_inds, conds,
                         dthreshold=5e-5, athreshold=0.02, w1=3.05, w2=1.0, times=5,
                         return_counters=False, mode="auto"):
    """OptimizeSurfacePs (utils/FindSurfacePs.py:114-163): returns (points, converged).
    Nothing syncs the host.  mode: "tc" = dense layers on the tensor-core engine (wgmma split-BF16,
    reverse-mode sweeps), "reverse" / "forward" = fused fp32 FFMA engine (times+1 launches of one
    persistent kernel), "auto" = "tc" for large ray sets, "reverse" otherwise."""
    if mode == "auto":
        mode = "tc" if (TC_ENABLED and init_pts.shape[0] >= TC_MIN_POINTS) else "reverse"
    if mode == "tc":
        return trace_surface_points_tc(sdf_net, def_net, lbs, cam_pos, rays, init_pts, batch_inds, conds,
                                       dthreshold, athreshold, w1, w2, times, return_counters)
    _need_cuda(rays, init_pts)
    dev = init_pts.device
    P = init_pts.shape[0]
    pts = init_pts.detach().contiguous().float().clone()
    rays = rays.detach().contiguous().float()
    bi = batch_inds.contiguous().to(torch.int64) if batch_inds is not None else None
    conds = conds.detach().contiguous().float() if conds is not None else None
    condlen = conds.shape[-1] if conds is not None else 0
    conv = torch.zeros((P,), dtype=torch.bool, device=dev)
    if P == 0:
        return (pts, conv, torch.zeros((times + 3,), dtype=torch.int32, device=dev)) if return_counters \
            else (pts, conv)
    lists = [torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(2)]
    counters = torch.zeros((times + 3,), dtype=torch.int32, device=dev)
    tp = TraceParams()
    cp = _host_floats(cam_pos)
    for i in range(3):
        tp.cam_pos[i] = cp[i]
    tp.dthreshold, tp.athreshold, tp.w1, tp.w2 = float(dthreshold), float(athreshold), float(w1), float(w2)
    lib = _lib.load()
    dref = C.byref(def_net.desc) if def_net is not None else None
    with torch.cuda.device(dev):
        scratch = _trace_scratch(dev) if mode == "reverse" else None
        for it in range(times + 1):
            a_in = lists[(it + 1) & 1] if it > 0 else None
            a_out = lists[it & 1] if it < times else None
            if mode == "reverse":
                check(lib.sr_trace_step_rev(C.byref(sdf_net.desc), dref, _lbs_ref(lbs), C.byref(tp),
                                            _p(pts), _p(rays), _p(bi), _p(conds), condlen, P, _p(a_in),
                                            _p(a_out), _p(counters), it, _p(conv), _p(scratch),
                                            _stream()), "trace_step_rev")
            else:
                check(lib.sr_trace_step(C.byref(sdf_net.desc), dref, _lbs_ref(lbs), C.byref(tp),
                                        _p(pts), _p(rays), _p(bi), _p(conds), condlen, P, _p(a_in),
                                        _p(a_out), _p(counters), it, _p(conv), _stream()),
                      "trace_step")
    if return_counters:  # counters[it] = rays updated in iteration it (it = 1..times)
        return pts, conv, counters
    return pts, conv


def shade_geometry(sdf_net, def_net, lbs, pts, rays, batch_inds, conds, nfeat=0, want_dpos=False):
    _need_cuda(pts, rays)
    dev = pts.device
    P = pts.shape[0]
    pts = pts.detach().contiguous().float()
    rays = rays.detach().contiguous().float()
    bi = batch_inds.contiguous().to(torch.int64) if batch_inds is not None else None
    conds = conds.detach().contiguous().float() if conds is not None else None
    condlen = conds.shape[-1] if conds is not None else 0
    normals = torch.empty((P, 3), dtype=torch.float32, device=dev)
    crays = torch.empty((P, 3), dtype=torch.float32, device=dev)
    feat = torch.empty((P, nfeat), dtype=torch.float32, device=dev) if nfeat else None
    dpos = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_dpos else None
    ok = torch.empty((P,), dtype=torch.bool, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        check(lib.sr_shade_geometry(C.byref(sdf_net.desc),
                                    C.byref(def_net.desc) if def_net is not None else None, _lbs_ref(lbs),
                                    _p(pts), _p(rays), _p(bi), _p(conds), condlen, P, _p(normals),
                                    _p(crays), _p(feat), int(nfeat), _p(dpos), _p(ok), _stream()),
              "shade_geometry")
    return normals, crays, feat, dpos, ok


# ------------------------------------------------------------------------------------------------
# Seg3dLossless plumbing
# ------------------------------------------------------------------------------------------------
def seg3d_candidates(flag, calculated, stride_zyx):
    """flag [D,H,W] bool, calculated [fD,fH,fW] bool -> candidate mask [D,H,W] bool."""
    _need_cuda(flag, calculated)
    D, H, W = flag.shape
    fD, fH, fW = calculated.shape
    cand = torch.empty((D, H, W), dtype=torch.bool, device=flag.device)
    lib = _lib.load()
    with torch.cuda.device(flag.device):
        check(lib.sr_seg3d_candidates(_p(flag.contiguous()), _p(calculated), _p(cand), D, H, W,
                                      int(stride_zyx[0]), int(stride_zyx[1]), int(stride_zyx[2]),
                                      fD, fH, fW, _stream()), "seg3d_candidates")
    return cand


_KERNELS_PER_CALL.update({"seg3d_candidates": 2, "seg3d_scatter": 3})


def seg3d_gather(lin, level_hw, stride_zyx, calculated, bmin, bmax, grid_flat):
    """lin [n] int64 (ids on the level lattice) -> (world points [n,3], interpolated values [n]);
    marks the points in `calculated` (final-grid bool mask).  bmin / bmax: python float triples."""
    _need_cuda(lin, calculated, grid_flat)
    n = lin.numel()
    dev = lin.device
    fD, fH, fW = calculated.shape
    pts = torch.empty((n, 3), dtype=torch.float32, device=dev)
    interp = torch.empty((n,), dtype=torch.float32, device=dev)
    lib = _lib.load()
    lo = (C.c_float * 3)(*[float(v) for v in bmin])
    hi = (C.c_float * 3)(*[float(v) for v in bmax])
    with torch.cuda.device(dev):
        check(lib.sr_seg3d_gather(_p(lin), n, int(level_hw[0]), int(level_hw[1]), int(stride_zyx[0]),
                                  int(stride_zyx[1]), int(stride_zyx[2]), fD, fH, fW, lo, hi, _p(grid_flat),
                                  _p(pts), _p(interp), _p(calculated), _stream()), "seg3d_gather")
    return pts, interp


def seg3d_scatter(lin, values, interp, balance, grid_flat):
    """grid[lin] = values; returns (conflict mask [numel(grid)] bool, n_conflicts int32[1] on device)."""
    _need_cuda(lin, values, interp, grid_flat)
    dev = lin.device
    conflict = torch.empty((grid_flat.numel(),), dtype=torch.bool, device=dev)
    ncf = torch.empty((1,), dtype=torch.int32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        check(lib.sr_seg3d_scatter(_p(lin), lin.numel(), _p(values), _p(interp), float(balance), _p(grid_flat),
                                   _p(conflict), conflict.numel(), _p(ncf), _stream()), "seg3d_scatter")
    return conflict, ncf


# ------------------------------------------------------------------------------------------------
# Tensor-core (wgmma, split-BF16) layer engine
# ------------------------------------------------------------------------------------------------
def tc_pack_rows(x):
    """fp32 [M,K] -> tiled split-bf16 activation buffer (uint8 tensor)."""
    _need_cuda(x)
    x = x.contiguous().float()
    M, K = x.shape
    lib = _lib.load()
    buf = torch.empty((lib.sr_tc_act_bytes(M, K),), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.sr_tc_pack_rows(_p(x), M, K, K, _p(buf), None, _stream()), "tc_pack_rows")
    return buf


def tc_pack_weights(w):
    """effective weights fp32 [N,K] -> tiled split-bf16 weight buffer (uint8 tensor)."""
    _need_cuda(w)
    w = w.contiguous().float()
    N, K = w.shape
    lib = _lib.load()
    buf = torch.empty((lib.sr_tc_weight_bytes(N, K),), dtype=torch.uint8, device=w.device)
    with torch.cuda.device(w.device):
        check(lib.sr_tc_pack_weights(_p(w), N, K, K, _p(buf), _stream()), "tc_pack_weights")
    return buf


def tc_linear(A, W, bias, M, N, K, n_valid, act, ch=1, K_next=0, scale=1.0, skip_src=None, skip_n=0,
              want_out=False):
    """One layer on the tensor-core engine.  Returns (A_next | None, out | None, None); the last slot, where an act'
    stash could be returned, stays None."""
    lib = _lib.load()
    dev = A.device
    A_next = torch.empty((lib.sr_tc_act_bytes(M, K_next),), dtype=torch.uint8, device=dev) if K_next else None
    out = torch.empty((M, n_valid), dtype=torch.float32, device=dev) if want_out else None
    npad = (N + 255) // 256 * 256
    b = torch.zeros((npad,), dtype=torch.float32, device=dev)
    b[:bias.numel()] = bias.reshape(-1)
    with torch.cuda.device(dev):
        check(lib.sr_tc_linear(_p(A), _p(W), _p(b), M, N, K, n_valid, int(act), int(ch), _p(A_next),
                               int(K_next), float(scale), _p(skip_src), int(skip_n),
                               skip_src.shape[1] if skip_src is not None else 0, _p(out),
                               n_valid if want_out else 0, 0, n_valid, None, None, 0, 0, 1.0, None, _stream()),
              "tc_linear")
    return A_next, out, None


class TcNet:
    """Tensor-core view of a FusedMLP: the same folded weights packed as tiled split-bf16 operands -- `W` for the
    forward sweep, `Wb` (= W^T) for the reverse sweep.  The pack buffers are persistent: `repack()` rewrites them
    in place when the FusedMLP is refolded, so launches recorded in a CUDA graph keep reading current weights."""

    def __init__(self, fused):
        self.fused = fused
        d = fused.desc
        self.layers = []
        lib = _lib.load()
        dev = fused.device
        for i in range(d.n_layers):
            ly = d.layer[i]
            e = fused._lay[i]
            n, k = ly.n, ly.k
            W = torch.empty((lib.sr_tc_weight_bytes(n, k),), dtype=torch.uint8, device=dev)
            Wb = torch.empty((lib.sr_tc_weight_bytes(k, n),), dtype=torch.uint8, device=dev)
            self.layers.append(dict(W=W, Wb=Wb, bias=torch.zeros((_pad(n, 256),), dtype=torch.float32, device=dev),
                                    n=n, k=k, act=ly.act, skip=bool(ly.skip), _e=e,
                                    zero_bias=torch.zeros((_pad(k, 256),), dtype=torch.float32, device=dev)))
        # the same packs as sr_tc_mlp_forward's layer array (repack() keeps the buffers, so the pointers stay valid)
        self.c_layers = (_lib.TcLayer * len(self.layers))()
        for c, L in zip(self.c_layers, self.layers):
            c.W, c.Wb, c.bias, c.zero_bias = (L[t].data_ptr() for t in ("W", "Wb", "bias", "zero_bias"))
            c.n, c.k, c.act, c.skip = L["n"], L["k"], L["act"], int(L["skip"])
        self.repack()

    def repack(self):
        lib = _lib.load()
        with torch.cuda.device(self.fused.device):
            for L in self.layers:
                e, n, k = L["_e"], L["n"], L["k"]
                check(lib.sr_tc_pack_weights(_p(e["wb"]), n, k, e["wb"].shape[1], _p(L["W"]), _stream()),
                      "tc_pack_weights")
                # reverse sweep operand: W^T as [k rows][n cols] = the FFMA engine's W_T copy (ld = npad)
                check(lib.sr_tc_pack_weights(_p(e["wt"]), k, n, e["wt"].shape[1], _p(L["Wb"]), _stream()),
                      "tc_pack_weights")
                L["bias"][:n].copy_(e["bias"][:n])


def tc_net(fused):
    t = getattr(fused, "_tc", None)
    if t is None:
        t = TcNet(fused)
        fused._tc = t
    return t


def _tc_mlp(lib, tcn, x0, ch, out, A_in=None, acts=None, m_dev=None):
    """Embedded input rows x0 fp32 [M][ld] -> the last layer's first out.shape[1] columns in `out` (one pack, then one
    wgmma launch per layer).  A_in / acts receive the input tiles and every hidden layer's output tiles when the caller
    keeps them (the tracer's reverse sweep recomputes act' from them); m_dev: optional device-side row count."""
    global LAUNCHES
    M, ld = x0.shape
    L = len(tcn.layers)
    if A_in is None:
        A_in = torch.empty((lib.sr_tc_act_bytes(M, ld),), dtype=torch.uint8, device=x0.device)
        acts = [torch.empty((lib.sr_tc_act_bytes(M, _pad(ly["k"], 32)),), dtype=torch.uint8, device=x0.device)
                for ly in tcn.layers[1:]]
    acts_c = (C.c_void_p * max(L - 1, 1))(*[a.data_ptr() for a in acts])
    check(lib.sr_tc_mlp_forward(tcn.c_layers, L, _p(x0), M, ld, tcn.fused.desc.d_in, ch, _p(A_in), acts_c, None,
                                _p(out), _p(m_dev), out.shape[1], _stream()), "tc_mlp_forward")
    LAUNCHES += L      # check() counted one; the call is 1 + L launches


def tc_mlp_forward(fused, pts, ch=1, conds=None, batch_inds=None, pts_per_frame=0, n_out=None):
    """Whole MLP on the tensor-core engine: embed -> pack -> one wgmma launch per layer.
    Returns out fp32 [P*ch, n_out] (last-layer outputs; tangent rows hold d out / d p_t)."""
    _need_cuda(pts)
    net = tc_net(fused)
    d = fused.desc
    dev = pts.device
    pts = pts.contiguous().float().view(-1, 3)
    P = pts.shape[0]
    M = P * ch
    condlen = conds.shape[-1] if conds is not None else 0
    ld = _pad(d.d_in, 32)
    lib = _lib.load()
    emb = torch.empty((M, ld), dtype=torch.float32, device=dev)
    out = torch.empty((M, n_out or net.layers[-1]["n"]), dtype=torch.float32, device=dev)
    pw = (C.c_float * 16)(*[d.pe_w[i] for i in range(16)])
    bi = batch_inds.contiguous().to(torch.int64) if batch_inds is not None else None
    cd = conds.detach().contiguous().float() if conds is not None else None
    with torch.cuda.device(dev):
        check(lib.sr_tc_embed(_p(pts), P, d.multires, pw, ch, _p(cd), _p(bi), int(pts_per_frame), condlen,
                              _p(emb), ld, None, None, _stream()), "tc_embed")
        _tc_mlp(lib, net, emb, ch, out)
    return out


class _TcTraceBuffers:
    """Work buffers of the tensor-core tracer, sized by the ray count and cached per device."""

    def __init__(self, dev, P, sdf_net, def_net):
        lib = _lib.load()
        self.P = P
        f32 = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
        u8 = lambda n: torch.empty((n,), dtype=torch.uint8, device=dev)
        self.ld_s = _pad(sdf_net.desc.d_in, 32)
        self.emb_s = f32(P, self.ld_s)
        # reverse-sweep staging tiles (ping-pong pair), as wide as the widest cotangent of either network
        widest = max([32] + [_pad(net.desc.layer[l].n, 32) for net in (sdf_net, def_net) if net is not None
                             for l in range(net.desc.n_layers - 1)])
        self.A = [u8(lib.sr_tc_act_bytes(P, widest)) for _ in range(2)]
        self.f = f32(P, 1)
        self.A_in = u8(lib.sr_tc_act_bytes(P, 256))
        self.acts_s = [u8(lib.sr_tc_act_bytes(P, _pad(sdf_net.desc.layer[i + 1].k, 32)))
                       for i in range(sdf_net.desc.n_layers - 1)]
        self.cot_s = f32(P, 32)
        self.cot_d = f32(P, 32)
        self.aux = f32(P, 8)
        self.gs = f32(P, 64)
        self.gskip = f32(P, 64)
        if def_net is not None:
            self.ld_d = _pad(def_net.desc.d_in, 32)
            self.emb_d = f32(P, self.ld_d)
            self.off = f32(P, 3)
            self.acts_d = [u8(lib.sr_tc_act_bytes(P, _pad(def_net.desc.layer[i + 1].k, 32)))
                           for i in range(def_net.desc.n_layers - 1)]
            self.gd = f32(P, 64)
            # the translator's sweeps run on a second stream beside the SDF's (own staging buffers)
            self.A_in_d = u8(lib.sr_tc_act_bytes(P, 256))
            self.A_d = [u8(lib.sr_tc_act_bytes(P, widest)) for _ in range(2)]
            self.gskip_d = f32(P, 64)


def _tc_backward_sweep(lib, tcn, cot, bufs, acts, P, m_dev, g_out, g_skip, n_keep):
    """cotangent rows `cot` [P][32] of the net outputs -> d/d(embedded input) in g_out [P][ld]
    (first n_keep columns), skip-connection part in g_skip.  acts = the forward sweep's tiles; bufs = a pair of
    staging tile buffers the layers alternate between."""
    d_in = tcn.fused.desc.d_in
    cur, nxt = bufs
    check(lib.sr_tc_pack_rows(_p(cot), P, 32, 32, _p(cur), _p(m_dev), _stream()), "tc_pack_rows")
    K = 32
    for l in range(len(tcn.layers) - 1, -1, -1):
        ly = tcn.layers[l]
        scale = 0.7071067811865476 if ly["skip"] else 1.0
        if l > 0:
            n_prev = tcn.layers[l - 1]["n"]
            Kn = _pad(n_prev, 32)
            gk = g_skip if ly["skip"] else None
            check(lib.sr_tc_linear(_p(cur), _p(ly["Wb"]), _p(ly["zero_bias"]), P, ly["k"], K, n_prev, 0, 1, _p(nxt),
                                   Kn, scale, None, 0, 0, _p(gk), gk.shape[1] if gk is not None else 0, n_prev,
                                   d_in if gk is not None else 0, None, _p(acts[l - 1]), _pad(ly["k"], 32),
                                   tcn.layers[l - 1]["act"], scale, _p(m_dev), _stream()), "tc_linear")
            cur, nxt, K = nxt, cur, Kn
        else:
            check(lib.sr_tc_linear(_p(cur), _p(ly["Wb"]), _p(ly["zero_bias"]), P, ly["k"], K, ly["k"], 0, 1, None, 0,
                                   scale, None, 0, 0, _p(g_out), g_out.shape[1], 0, n_keep, None, None, 0, 0, 1.0,
                                   _p(m_dev), _stream()), "tc_linear")


class _TcTraceCtx:
    """Static state of one tensor-core trace configuration: work buffers, static input / output
    tensors and (after the second call) the captured CUDA graph of the whole trace.  Everything a
    launch reads through a pointer lives here, so a replay only needs fresh contents copied in."""

    def __init__(self, dev, P, sdf_net, def_net, n_frames, condlen, times):
        self.B = _TcTraceBuffers(dev, P, sdf_net, def_net)
        self.pts = torch.empty((P, 3), dtype=torch.float32, device=dev)
        self.rays = torch.empty((P, 3), dtype=torch.float32, device=dev)
        self.bi = torch.empty((P,), dtype=torch.int64, device=dev)
        self.conds = torch.empty((n_frames, condlen), dtype=torch.float32, device=dev) if condlen else None
        self.conv = torch.empty((P,), dtype=torch.bool, device=dev)
        self.counters = torch.empty((times + 3,), dtype=torch.int32, device=dev)
        self.lists = [torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(2)]
        self.lbsA = torch.empty((n_frames, 24, 4, 4), dtype=torch.float32, device=dev)
        self.lbsT = torch.empty((n_frames, 3), dtype=torch.float32, device=dev)
        self.lbs_params = LbsParams()
        # borderline rays of each iteration, re-tested on the fp32 engine (one list, one count per iteration)
        self.side_stream = torch.cuda.Stream(device=dev)
        self.recheck = torch.empty((P,), dtype=torch.int32, device=dev)
        self.recheck_counts = torch.empty((times + 1,), dtype=torch.int32, device=dev)
        self.rev_scratch = _trace_scratch(dev)
        self.graph = None
        self.sig = None
        self.calls = 0
        self.n_launches = 0


_tc_trace_ctx = {}
GRAPHS_ENABLED = _os.environ.get("SELFRECON_B200_GRAPHS", "1") != "0"


def _tc_trace_body(lib, G, sdf_net, def_net, ts, td, tp, P, times, condlen, has_lbs):
    """All launches of one trace on the current stream (eager, or under CUDA-graph capture)."""
    B = G.B
    ds, dd = sdf_net.desc, (def_net.desc if def_net is not None else None)
    pw_s = (C.c_float * 16)(*[ds.pe_w[i] for i in range(16)])
    pw_d = (C.c_float * 16)(*[dd.pe_w[i] for i in range(16)]) if dd is not None else None
    pts, rays, bi, conds, conv, counters, lists = G.pts, G.rays, G.bi, G.conds, G.conv, G.counters, G.lists
    lbs_ref = C.byref(G.lbs_params) if has_lbs else None
    conv.zero_()
    counters.zero_()
    counters[0:1].fill_(P)
    refine = TC_REFINE_TRACE
    if refine:
        G.recheck_counts.zero_()
    dref = C.byref(def_net.desc) if def_net is not None else None
    for it in range(times + 1):
        idx = lists[(it + 1) & 1] if it > 0 else None
        a_out = lists[it & 1] if it < times else None
        m_dev = counters[it:it + 1]
        # ---- forward sweeps (each layer keeps its output tiles for the reverse sweep)
        check(lib.sr_tc_embed(_p(pts), P, ds.multires, pw_s, 1, None, None, 0, 0, _p(B.emb_s), B.ld_s,
                              _p(idx), _p(m_dev), _stream()), "tc_embed")
        # The SDF sweep (9 launches) and the translator sweep (5 launches) of an iteration are independent: on two
        # streams the second grid's CTAs move into the SMs the first grid's last wave leaves idle (5.3 waves of row
        # tiles per launch at 50 333 rays) and into its ramp / tail, instead of waiting for the whole grid.
        dual = TC_DUAL_STREAM and def_net is not None
        if dual:
            main = torch.cuda.current_stream()
            side = G.side_stream
            side.wait_stream(main)
            with torch.cuda.stream(side):
                check(lib.sr_tc_embed(_p(pts), P, dd.multires, pw_d, 1, _p(conds), _p(bi), 0, condlen,
                                      _p(B.emb_d), B.ld_d, _p(idx), _p(m_dev), _stream()), "tc_embed")
                _tc_mlp(lib, td, B.emb_d, 1, B.off, B.A_in_d, B.acts_d, m_dev)
        _tc_mlp(lib, ts, B.emb_s, 1, B.f, B.A_in, B.acts_s, m_dev)
        if dual:
            main.wait_stream(side)
        elif def_net is not None:
            check(lib.sr_tc_embed(_p(pts), P, dd.multires, pw_d, 1, _p(conds), _p(bi), 0, condlen,
                                  _p(B.emb_d), B.ld_d, _p(idx), _p(m_dev), _stream()), "tc_embed")
            _tc_mlp(lib, td, B.emb_d, 1, B.off, B.A_in, B.acts_d, m_dev)
        check(lib.sr_tc_trace_mid(_p(idx), _p(m_dev), P, _p(pts), _p(rays), _p(bi), _p(B.f),
                                  _p(B.off) if def_net is not None else None, lbs_ref, C.byref(tp),
                                  1 if a_out is not None else 0, _p(conv), _p(B.cot_s),
                                  _p(B.cot_d) if def_net is not None else None, 32, _p(B.aux),
                                  _p(G.recheck) if refine else None,
                                  _p(G.recheck_counts[it:it + 1]) if refine else None,
                                  TC_EPS_F if refine else 0.0, TC_EPS_A if refine else 0.0, _stream()),
              "tc_trace_mid")
        if refine:
            # fp32 re-test of the borderline rays (test-only launch: no update, marks converged[])
            check(lib.sr_trace_step_rev(C.byref(sdf_net.desc), dref, lbs_ref, C.byref(tp), _p(pts), _p(rays),
                                        _p(bi), _p(conds), condlen, P, _p(G.recheck), None,
                                        _p(G.recheck_counts), it, _p(conv), _p(G.rev_scratch), _stream()),
                  "trace_step_rev")
        if a_out is None:
            break
        # ---- reverse sweeps + update
        if dual:
            side.wait_stream(main)
            with torch.cuda.stream(side):
                _tc_backward_sweep(lib, td, B.cot_d, B.A_d, B.acts_d, P, m_dev, B.gd, B.gskip_d, 3 + 6 * dd.multires)
        _tc_backward_sweep(lib, ts, B.cot_s, B.A, B.acts_s, P, m_dev, B.gs, B.gskip, ds.d_in)
        if dual:
            main.wait_stream(side)
        elif def_net is not None:
            _tc_backward_sweep(lib, td, B.cot_d, B.A, B.acts_d, P, m_dev, B.gd, B.gskip, 3 + 6 * dd.multires)
        has_skip = any(l["skip"] for l in ts.layers)
        check(lib.sr_tc_trace_update(_p(idx), _p(m_dev), P, _p(pts), _p(B.gs), B.gs.shape[1],
                                     _p(B.gskip) if has_skip else None, B.gskip.shape[1],
                                     _p(B.gd) if def_net is not None else None,
                                     B.gd.shape[1] if def_net is not None else 0, _p(B.aux), ds.multires,
                                     pw_s, dd.multires if dd is not None else 0, pw_d, _p(a_out),
                                     _p(counters[it + 1:it + 2]), _p(conv) if refine else None, _stream()),
              "tc_trace_update")


def trace_surface_points_tc(sdf_net, def_net, lbs, cam_pos, rays, init_pts, batch_inds, conds,
                            dthreshold=5e-5, athreshold=0.02, w1=3.05, w2=1.0, times=5,
                            return_counters=False):
    """OptimizeSurfacePs with the dense layers on the tensor-core engine (reverse-mode sweeps).
    Same contract as trace_surface_points.  A trace is ~35 launches per iteration, all with static
    shapes and device-side counts, so from the second call with the same configuration (ray count,
    networks, thresholds, PE weights) the whole trace is replayed as one CUDA graph
    (SELFRECON_B200_GRAPHS=0 keeps it eager)."""
    global LAUNCHES
    _need_cuda(rays, init_pts)
    dev = init_pts.device
    P = init_pts.shape[0]
    if P == 0:
        pts = init_pts.detach().float().clone()
        conv = torch.zeros((0,), dtype=torch.bool, device=dev)
        return (pts, conv, torch.zeros((times + 3,), dtype=torch.int32, device=dev)) if return_counters \
            else (pts, conv)
    lib = _lib.load()
    condlen = conds.shape[-1] if conds is not None else 0
    n_frames = lbs.A.shape[0] if lbs is not None else (conds.shape[0] if conds is not None else 1)
    cp = _host_floats(cam_pos)
    ds, dd = sdf_net.desc, (def_net.desc if def_net is not None else None)
    # buffers depend on shapes only; the captured graph also on everything a launch bakes in
    key = (dev.index, P, tuple(ds.layer[i].n for i in range(ds.n_layers)),
           tuple(dd.layer[i].n for i in range(dd.n_layers)) if dd is not None else (), n_frames, condlen,
           conds.shape[0] if conds is not None else 0, times)
    sig = (sdf_net.uid, def_net.uid if def_net is not None else -1,
           lbs.ws_cl.data_ptr() if lbs is not None else 0, cp, float(dthreshold), float(athreshold),
           float(w1), float(w2), tuple(ds.pe_w[i] for i in range(ds.multires)),
           tuple(dd.pe_w[i] for i in range(dd.multires)) if dd is not None else (),
           TC_REFINE_TRACE, TC_EPS_F, TC_EPS_A, TC_DUAL_STREAM)
    G = _tc_trace_ctx.get(key)
    if G is None:
        if len(_tc_trace_ctx) >= 4:
            _tc_trace_ctx.pop(next(iter(_tc_trace_ctx)))
        G = _TcTraceCtx(dev, P, sdf_net, def_net, n_frames, condlen, times)
        _tc_trace_ctx[key] = G
    if G.sig != sig:          # new weights / thresholds: the old graph is stale, buffers are not
        G.sig, G.graph, G.calls = sig, None, 0
    ts, td = tc_net(sdf_net), (tc_net(def_net) if def_net is not None else None)
    tp = TraceParams()
    for i in range(3):
        tp.cam_pos[i] = cp[i]
    tp.dthreshold, tp.athreshold, tp.w1, tp.w2 = float(dthreshold), float(athreshold), float(w1), float(w2)
    with torch.cuda.device(dev):
        G.pts.copy_(init_pts.detach().reshape(P, 3))
        G.rays.copy_(rays.detach().reshape(P, 3))
        if batch_inds is not None:
            G.bi.copy_(batch_inds.reshape(P))
        else:
            G.bi.zero_()
        if conds is not None:
            G.conds.copy_(conds.detach())
        if lbs is not None:
            G.lbsA.copy_(lbs.A)
            G.lbsT.copy_(lbs.trans)
            C.memmove(C.byref(G.lbs_params), C.byref(lbs.params), C.sizeof(LbsParams))
            G.lbs_params.A = G.lbsA.data_ptr()
            G.lbs_params.trans = G.lbsT.data_ptr()
        args = (lib, G, sdf_net, def_net, ts, td, tp, P, times, condlen, lbs is not None)
        if G.graph is not None:
            G.graph.replay()
            LAUNCHES += G.n_launches
        elif GRAPHS_ENABLED and G.calls >= 1:
            before = LAUNCHES
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                _tc_trace_body(*args)
            G.n_launches = LAUNCHES - before
            G.graph = g
            g.replay()
        else:
            _tc_trace_body(*args)
        G.calls += 1
        out = (G.pts.clone(), G.conv.clone())
        if return_counters:
            out = out + (G.counters.clone(),)
    return out


_side_streams = {}


def _side_stream(dev):
    st = _side_streams.get(dev.index)
    if st is None:
        st = torch.cuda.Stream(device=dev)
        _side_streams[dev.index] = st
    return st


def shade_and_render_tc(sdf_full, def_net, lbs, render_net, pts, rays, batch_inds, conds, nfeat=256):
    """Shading of the infer path on the tensor-core engine: SDF and translator sweeps with forward
    tangents (4 rows per point), pointwise geometry, then the rendering network.
    Returns (normals, cardinal rays, rgb, D(p), inverse-ok mask)."""
    _need_cuda(pts, rays)
    dev = pts.device
    P = pts.shape[0]
    pts = pts.detach().contiguous().float()
    rays = rays.detach().contiguous().float()
    bi = batch_inds.contiguous().to(torch.int64) if batch_inds is not None else None
    lib = _lib.load()
    with torch.cuda.device(dev):
        if TC_DUAL_STREAM and def_net is not None:
            # SDF and translator sweeps are independent: second stream (see _tc_trace_body)
            main = torch.cuda.current_stream()
            side = _side_stream(dev)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                o4 = tc_mlp_forward(def_net, pts, ch=4, conds=conds, batch_inds=bi)
            s4 = tc_mlp_forward(sdf_full, pts, ch=4)                  # [4P, 1+nfeat]
            main.wait_stream(side)
            o4.record_stream(main)
        else:
            s4 = tc_mlp_forward(sdf_full, pts, ch=4)
            o4 = tc_mlp_forward(def_net, pts, ch=4, conds=conds, batch_inds=bi) if def_net is not None else None
        normals = torch.empty((P, 3), dtype=torch.float32, device=dev)
        crays = torch.empty((P, 3), dtype=torch.float32, device=dev)
        dpos = torch.empty((P, 3), dtype=torch.float32, device=dev)
        ok = torch.empty((P,), dtype=torch.bool, device=dev)
        check(lib.sr_tc_shade_point(P, _p(pts), _p(rays), _p(bi), _p(s4), s4.shape[1], _p(o4), _lbs_ref(lbs),
                                    _p(normals), _p(crays), _p(dpos), _p(ok), _stream()), "tc_shade_point")
        rd = render_net.desc
        ld = _pad(rd.d_in, 32)
        emb = torch.empty((P, ld), dtype=torch.float32, device=dev)
        pw = (C.c_float * 16)(*[rd.pe_w[i] for i in range(16)])
        check(lib.sr_tc_render_embed(P, _p(pts), _p(crays), _p(normals), _p(s4), s4.shape[1], 1, nfeat, 4,
                                     rd.multires, pw, _p(emb), ld, _stream()), "tc_render_embed")
        rn = tc_net(render_net)
        rgb = torch.empty((P, rn.layers[-1]["n"]), dtype=torch.float32, device=dev)
        _tc_mlp(lib, rn, emb, 1, rgb)
    return normals, crays, rgb, dpos, ok
