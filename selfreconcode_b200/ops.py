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

# The tensor-core engine's error bound (DESIGN.md section 4): TC_EPS_F bounds its absolute error on an SDF value
# (split-BF16 with fp32 accumulation, csrc/tc_gemm.cu), and sign decisions inside it are re-taken on the fp32 FFMA
# engine (sdf_refine_band).
TC_EPS_F = 4e-5
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
    if N == 0 or F == 0:
        # no frame, or a mesh without faces: every pixel is background (the kernels refuse empty inputs)
        return (torch.full((N, H, W, 1), -1, dtype=torch.int64, device=dev),
                torch.full((N, H, W, 1, 3), -1., dtype=torch.float32, device=dev),
                torch.full((N, H, W, 1), -1., dtype=torch.float32, device=dev))
    keys = torch.empty((N, H, W), dtype=torch.int64, device=dev)
    p2f = torch.empty((N, H, W, 1), dtype=torch.int64, device=dev)
    bary = torch.empty((N, H, W, 1, 3), dtype=torch.float32, device=dev)
    zbuf = torch.empty((N, H, W, 1), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().sr_raster_mesh(_p(vs), _p(fc), N, V, F, int(H), int(W), _p(keys), _p(p2f), _p(bary),
                                         _p(zbuf), _stream()), "raster_mesh")
    return p2f, bary, zbuf


_KERNELS_PER_CALL["raster_mesh"] = 2


def mesh_vertex_normals(verts, faces, csr):
    """verts [N,V,3] world positions of N frames sharing faces [F,3] int64; csr = (offsets [V+1], face ids) of each
    vertex's incident faces, ascending -> [N,V,3] pytorch3d vertex normals (area-weighted, F.normalize eps 1e-6)."""
    _need_cuda(verts, faces, csr[0], csr[1])
    vs = verts.detach().contiguous().float()
    fc = faces.contiguous().to(torch.int64)
    off, fid = csr[0].contiguous().to(torch.int64), csr[1].contiguous().to(torch.int64)
    N, V, _ = vs.shape
    if off.numel() != V + 1:
        raise ValueError("mesh_vertex_normals: csr offsets must have V + 1 entries")
    out = torch.empty_like(vs)
    with torch.cuda.device(vs.device):
        check(_lib.load().sr_mesh_vertex_normals(_p(vs), _p(fc), _p(off), _p(fid), N, V, fc.shape[0], _p(out),
                                                 _stream()), "mesh_vertex_normals")
    return out


def shade_phong(verts, normals, faces, pix_to_face, bary, cam_pos, light_pos, params, colors=None):
    """pytorch3d HardPhongShader (phong_shading + hard_rgb_blend, one face per pixel) on rasteriser fragments.
    verts / normals / colors [N,V,3] (colors None = white), pix_to_face [N,H,W(,1)] packed ids, bary [N,H,W(,1),3],
    cam_pos / light_pos [N,3] device tensors, params a _lib.PhongParams -> images [N,H,W,4]."""
    _need_cuda(verts, normals, faces, pix_to_face, bary, cam_pos, light_pos, colors)
    vs = verts.detach().contiguous().float()
    N, V, _ = vs.shape
    H, W = pix_to_face.shape[1], pix_to_face.shape[2]
    nr = normals.detach().contiguous().float()
    col = colors.detach().contiguous().float() if colors is not None else None
    fc = faces.contiguous().to(torch.int64)
    p2f = pix_to_face.contiguous().to(torch.int64)
    br = bary.detach().contiguous().float()
    cp = cam_pos.detach().float().reshape(-1, 3).expand(N, 3).contiguous()
    lp = light_pos.detach().float().reshape(-1, 3).expand(N, 3).contiguous()
    if nr.shape != vs.shape or (col is not None and col.shape != vs.shape) or p2f.numel() != N * H * W \
            or br.numel() != 3 * N * H * W:
        raise ValueError("shade_phong: inconsistent shapes")
    out = torch.empty((N, H, W, 4), dtype=torch.float32, device=vs.device)
    with torch.cuda.device(vs.device):
        check(_lib.load().sr_shade_phong(_p(vs), _p(nr), _p(col), _p(fc), N, V, fc.shape[0], _p(p2f), _p(br),
                                         int(H), int(W), _p(cp), _p(lp), C.byref(params), _p(out), _stream()),
              "shade_phong")
    return out


_KERNELS_PER_CALL.update({"mesh_vertex_normals": 1, "shade_phong": 1})


POINTS_TILE = 16     # SR_POINTS_TILE: pixels per side of a tile of sr_points_silhouette_forward


class _PointsSilhouette(torch.autograd.Function):
    """Soft point silhouette (csrc/points_silhouette.cu): pytorch3d's PointsRasterizer + AlphaCompositor with unit
    features, differentiable w.r.t. the (col, row) screen coordinates."""

    @staticmethod
    def forward(ctx, pts_screen, H, W, radius, K):
        _need_cuda(pts_screen)
        vs = pts_screen.detach().contiguous().float()
        if vs.dim() != 3 or vs.shape[2] != 3:
            raise ValueError("points_silhouette: pts_screen must be [N,V,3]")
        N, V, _ = vs.shape
        lib = _lib.load()
        cap = lib.sr_points_silhouette_list_capacity(N, V, H, W, radius)
        if cap < 0:
            raise ValueError("points_silhouette: invalid sizes / radius (N=%d V=%d H=%d W=%d r=%r K=%d)"
                             % (N, V, H, W, radius, K))
        if K <= 0:
            raise ValueError("points_silhouette: points_per_pixel must be positive")
        dev = vs.device
        tiles = ((H + POINTS_TILE - 1) // POINTS_TILE) * ((W + POINTS_TILE - 1) // POINTS_TILE)
        with torch.cuda.device(dev):
            z = vs[..., 2]
            # each frame's points in (Z, index) order: a stable sort keeps equal depths in index order
            order = torch.sort(torch.where(z >= 0, z, torch.full_like(z, math.inf)), dim=1, stable=True).indices
            keys = torch.empty(cap, dtype=torch.int64, device=dev)
            ids = torch.empty(cap, dtype=torch.int32, device=dev)
            check(lib.sr_points_silhouette_bin(_p(vs), _p(order), N, V, H, W, radius, _p(keys), _p(ids), _stream()),
                  "points_silhouette_bin")
            keys, perm = torch.sort(keys, stable=True)       # tile-major, (Z, index) order kept inside each tile
            ids = ids[perm]
            offsets = torch.searchsorted(keys, torch.arange(N * tiles + 1, dtype=torch.int64, device=dev))
            mask = torch.empty((N, H, W, 1), dtype=torch.float32, device=dev)
            kth = torch.empty((N, H, W), dtype=torch.int64, device=dev)
            prod = torch.empty((N, H, W), dtype=torch.float32, device=dev)
            zeros = torch.empty((N, H, W), dtype=torch.int32, device=dev)
            check(lib.sr_points_silhouette_forward(_p(vs), _p(offsets), _p(ids), N, V, H, W, radius, K, _p(mask),
                                                   _p(kth), _p(prod), _p(zeros), _stream()),
                  "points_silhouette_forward")
        ctx.save_for_backward(vs, kth, prod, zeros)
        ctx.args = (H, W, radius)
        ctx.in_dtype = pts_screen.dtype
        return mask

    @staticmethod
    def backward(ctx, grad_mask):
        vs, kth, prod, zeros = ctx.saved_tensors
        H, W, radius = ctx.args
        N, V, _ = vs.shape
        g = grad_mask.contiguous().float()
        out = torch.empty_like(vs)
        with torch.cuda.device(vs.device):
            check(_lib.load().sr_points_silhouette_backward(_p(vs), _p(g), _p(kth), _p(prod), _p(zeros), N, V, H, W,
                                                            radius, _p(out), _stream()),
                  "points_silhouette_backward")
        return out.to(ctx.in_dtype), None, None, None, None


def points_silhouette(pts_screen, H, W, radius, K):
    """pts_screen [N,V,3] = (col, row, view-space Z) per frame (raster.screen_vertices), radius in NDC units,
    K points per pixel -> soft silhouette [N,H,W,1] (pytorch3d 0.4.0 PointsRasterizer + AlphaCompositor, unit
    features); differentiable w.r.t. (col, row).  DESIGN.md section 3.3."""
    return _PointsSilhouette.apply(pts_screen, int(H), int(W), float(radius), int(K))


_KERNELS_PER_CALL.update({"points_silhouette_bin": 1, "points_silhouette_forward": 1,
                          "points_silhouette_backward": 1})


MESH_REG_BLOCKS = 528     # SR_MESH_REG_BLOCKS


class MeshRegTopology:
    """Device tables of one face table for mesh_regularizers (csrc/mesh_reg.cu): the unique edges [E,2] in pytorch3d's
    order, face_to_edge [F,3], the directed neighbour CSR (nbr_off [V+1], nbr), the normal-consistency pairs [P,4] =
    (a, b, o_i, o_j) and the vertex -> (pair, role) CSR (vp_off [V+1], vp_ent = 4 pair + role)."""

    def __init__(self, V, F, E, P, edges, face_to_edge, nbr_off, nbr, pairs, vp_off, vp_ent):
        self.V, self.F, self.E, self.P = V, F, E, P
        self.edges, self.face_to_edge = edges, face_to_edge
        self.nbr_off, self.nbr = nbr_off, nbr
        self.pairs, self.vp_off, self.vp_ent = pairs, vp_off, vp_ent


def mesh_reg_topology(faces, V):
    """faces [F,3] int64 CUDA of a mesh with V vertices -> MeshRegTopology (pytorch3d 0.4.0 Meshes._compute_packed
    edges and mesh_normal_consistency pairs).  Reads E and P back to the host once; a face index outside [0, V) is a
    ValueError."""
    _need_cuda(faces)
    fc = faces.detach().contiguous().to(torch.int64)
    V = int(V)
    if fc.dim() != 2 or fc.shape[1] != 3 or fc.shape[0] == 0 or V <= 0:
        raise ValueError("mesh_reg_topology: faces must be [F,3] with F > 0 and V > 0")
    F = fc.shape[0]
    dev = fc.device
    lib = _lib.load()
    with torch.cuda.device(dev):
        keys = torch.empty(3 * F, dtype=torch.int64, device=dev)
        check(lib.sr_mesh_reg_edge_keys(_p(fc), F, V, _p(keys), _stream()), "mesh_reg_edge_keys")
        skeys, perm = torch.sort(keys, stable=True)     # unique edges ascending, (face, corner) order inside each
        head, npairs = torch.empty_like(skeys), torch.empty_like(skeys)
        check(lib.sr_mesh_reg_edge_runs(_p(skeys), 3 * F, _p(head), _p(npairs), _stream()), "mesh_reg_edge_runs")
        head_cum, pair_cum = torch.cumsum(head, 0), torch.cumsum(npairs, 0)
        bad, E, P = torch.stack([(skeys[0] < 0).long(), head_cum[-1], pair_cum[-1]]).tolist()
        if bad:
            raise ValueError("mesh_reg_topology: a face index is outside [0, %d)" % V)
        edges = torch.empty((E, 2), dtype=torch.int64, device=dev)
        f2e = torch.empty((F, 3), dtype=torch.int64, device=dev)
        dkeys = torch.empty(2 * E, dtype=torch.int64, device=dev)
        pairs = torch.empty((P, 4), dtype=torch.int64, device=dev)
        check(lib.sr_mesh_reg_topology(_p(fc), _p(skeys), _p(perm), _p(head_cum), _p(pair_cum), F, V, E, P,
                                       _p(edges), _p(f2e), _p(dkeys), _p(pairs if P else None), _stream()),
              "mesh_reg_topology")
        dkeys = torch.sort(dkeys).values
        nbr_off = torch.searchsorted(dkeys, torch.arange(V + 1, dtype=torch.int64, device=dev) * V)
        nbr = torch.remainder(dkeys, V)
        vid, vp_ent = torch.sort(pairs.reshape(-1), stable=True)
        vp_off = torch.searchsorted(vid, torch.arange(V + 1, dtype=torch.int64, device=dev))
    return MeshRegTopology(V, F, E, P, edges, f2e, nbr_off, nbr, pairs, vp_off, vp_ent)


class _MeshRegularizers(torch.autograd.Function):
    """(laplacian, edge, normal consistency) of one mesh (csrc/mesh_reg.cu), differentiable w.r.t. the vertices."""

    @staticmethod
    def forward(ctx, verts, topo):
        _need_cuda(verts)
        vs = verts.detach().contiguous().float()
        if tuple(vs.shape) != (topo.V, 3):
            raise ValueError("mesh_regularizers: verts must be [%d,3], got %s" % (topo.V, tuple(vs.shape)))
        dev = vs.device
        u = torch.empty((topo.V, 3), dtype=torch.float64, device=dev)
        dn = torch.empty((topo.P, 6), dtype=torch.float64, device=dev)
        part = torch.empty(3 * MESH_REG_BLOCKS, dtype=torch.float64, device=dev)
        out = torch.empty(3, dtype=torch.float32, device=dev)
        pairs = topo.pairs if topo.P else None
        with torch.cuda.device(dev):
            check(_lib.load().sr_mesh_reg_forward(_p(vs), topo.V, topo.E, topo.P, _p(topo.edges), _p(topo.nbr_off),
                                                  _p(topo.nbr), _p(pairs), _p(u), _p(dn if topo.P else None),
                                                  _p(part), _p(out), _stream()), "mesh_reg_forward")
        ctx.save_for_backward(vs, u, dn)
        ctx.topo = topo
        ctx.in_dtype = verts.dtype
        return out

    @staticmethod
    def backward(ctx, grad_out):
        vs, u, dn = ctx.saved_tensors
        topo = ctx.topo
        g = grad_out.contiguous().float()
        out = torch.empty_like(vs)
        has_p = topo.P > 0
        with torch.cuda.device(vs.device):
            check(_lib.load().sr_mesh_reg_backward(
                _p(vs), topo.V, topo.E, topo.P, _p(topo.nbr_off), _p(topo.nbr), _p(topo.pairs if has_p else None),
                _p(topo.vp_off), _p(topo.vp_ent if has_p else None), _p(u), _p(dn if has_p else None), _p(g),
                _p(out), _stream()), "mesh_reg_backward")
        return out.to(ctx.in_dtype), None


def mesh_regularizers(verts, topo):
    """verts [V,3] CUDA, topo = mesh_reg_topology(faces, V) -> [3] float32 = (mesh_laplacian_smoothing(method='uniform'),
    mesh_edge_loss(target_length=0.), mesh_normal_consistency) of pytorch3d 0.4.0 on one mesh; differentiable w.r.t.
    verts.  DESIGN.md section 3.3."""
    return _MeshRegularizers.apply(verts, topo)


_KERNELS_PER_CALL.update({"mesh_reg_edge_keys": 1, "mesh_reg_edge_runs": 1, "mesh_reg_topology": 1,
                          "mesh_reg_forward": 2, "mesh_reg_backward": 1})


def simplify_quadrics(verts, faces, csr, topo):
    """One simplification round's vertex pass (csrc/mesh_simplify.cu): verts [V,3] float32, faces [F,3] int64, csr =
    (offsets, face ids) of each vertex's faces, topo = mesh_reg_topology(faces, V) -> (Q [V,10] float64, fixed [V]
    uint8)."""
    _need_cuda(verts, faces, csr[0], csr[1])
    V, F = verts.shape[0], faces.shape[0]
    Q = torch.empty((V, 10), dtype=torch.float64, device=verts.device)
    fixed = torch.empty(V, dtype=torch.uint8, device=verts.device)
    with torch.cuda.device(verts.device):
        check(_lib.load().sr_simplify_quadrics(_p(verts), _p(faces), V, F, _p(csr[0]), _p(csr[1]), _p(topo.nbr_off),
                                               _p(topo.nbr), _p(Q), _p(fixed), _stream()), "simplify_quadrics")
    return Q, fixed


def simplify_edge_cost(verts, faces, csr, topo, Q, fixed):
    """-> (vstar [E,3] float64, cost [E] float64, key [E] int64 holding the uint64 keys: ~0 = -1 for an edge that may
    not collapse) of the edges topo.edges."""
    _need_cuda(verts, faces, Q, fixed)
    E, dev = topo.E, verts.device
    vstar = torch.empty((E, 3), dtype=torch.float64, device=dev)
    cost = torch.empty(E, dtype=torch.float64, device=dev)
    key = torch.empty(E, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().sr_simplify_edge_cost(_p(verts), _p(faces), _p(topo.edges), E, _p(csr[0]), _p(csr[1]),
                                                _p(topo.nbr_off), _p(topo.nbr), _p(Q), _p(fixed), _p(vstar), _p(cost),
                                                _p(key), _stream()), "simplify_edge_cost")
    return vstar, cost, key


def simplify_select(topo, key):
    """-> sel [E] uint8: the edges whose key is the minimum over the two rings of both endpoints."""
    _need_cuda(key)
    dev = key.device
    m1 = torch.empty(topo.V, dtype=torch.int64, device=dev)
    m2 = torch.empty_like(m1)
    sel = torch.empty(topo.E, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().sr_simplify_select(_p(topo.edges), topo.E, topo.V, _p(topo.nbr_off), _p(topo.nbr), _p(key),
                                             _p(m1), _p(m2), _p(sel), _stream()), "simplify_select")
    return sel


def simplify_collapse(verts, faces, edges, sel, vstar, n_verts, n_faces):
    """Collapses the selected edges (each removes one vertex and two faces) -> (verts [n_verts,3], faces [n_faces,3]),
    survivors in ascending order.  n_verts / n_faces are the counts the caller derived from its selection."""
    _need_cuda(verts, faces, edges, sel, vstar)
    V, F, E, dev = verts.shape[0], faces.shape[0], edges.shape[0], verts.device
    lib = _lib.load()
    remap = torch.empty(V, dtype=torch.int64, device=dev)
    pos = torch.empty_like(verts)
    face_alive = torch.empty(F, dtype=torch.uint8, device=dev)
    vert_alive = torch.empty(V, dtype=torch.uint8, device=dev)
    out_v = torch.empty((n_verts, 3), dtype=torch.float32, device=dev)
    out_f = torch.empty((n_faces, 3), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(lib.sr_simplify_collapse(_p(verts), _p(faces), V, F, _p(edges), E, _p(sel), _p(vstar), _p(remap),
                                       _p(pos), _p(face_alive), _p(vert_alive), _stream()), "simplify_collapse")
        face_cum, vert_cum = torch.cumsum(face_alive, 0), torch.cumsum(vert_alive, 0)
        check(lib.sr_simplify_compact(_p(faces), V, F, _p(remap), _p(pos), _p(face_alive), _p(vert_alive),
                                      _p(face_cum), _p(vert_cum), _p(out_v), _p(out_f), _stream()), "simplify_compact")
    return out_v, out_f


_KERNELS_PER_CALL.update({"simplify_select": 3, "simplify_collapse": 3})


def uv_face_adjacency(faces, csr):
    """faces [F,3] int64, csr = vertex -> face CSR -> adj [F,3] int64 (the face across each corner's opposite edge
    when that edge has two faces, else -1)."""
    _need_cuda(faces, csr[0], csr[1])
    F = faces.shape[0]
    adj = torch.empty((F, 3), dtype=torch.int64, device=faces.device)
    with torch.cuda.device(faces.device):
        check(_lib.load().sr_uv_face_adjacency(_p(faces), F, _p(csr[0]), _p(csr[1]), _p(adj), _stream()),
              "uv_face_adjacency")
    return adj


UV_DIRECTIONS = 26


def uv_labels(verts, faces, adj, max_angle, passes=8):
    """-> (unit normals [F,3] float64, areas [F] float64, labels [F] int32 in [0, 26)) after `passes` smoothing
    passes."""
    _need_cuda(verts, faces, adj)
    F, dev = faces.shape[0], verts.device
    normal = torch.empty((F, 3), dtype=torch.float64, device=dev)
    area = torch.empty(F, dtype=torch.float64, device=dev)
    label = torch.empty(F, dtype=torch.int32, device=dev)
    work = torch.empty_like(label)
    with torch.cuda.device(dev):
        check(_lib.load().sr_uv_labels(_p(verts), _p(faces), F, _p(adj), float(max_angle), int(passes), _p(normal),
                                       _p(area), _p(label), _p(work), _stream()), "uv_labels")
    return normal, area, label


_KERNELS_PER_CALL["uv_labels"] = 9


def uv_chart_ids(adj, label, check_every=8):
    """-> cid [F] int64 = the minimum face id of each face's chart (same-label faces joined across two-face edges).
    Hooking passes run in groups of check_every between readbacks of the changed flag."""
    _need_cuda(adj, label)
    F, dev = label.shape[0], label.device
    cid = torch.arange(F, dtype=torch.int64, device=dev)
    changed = torch.empty(1, dtype=torch.int32, device=dev)
    flags = torch.empty(check_every, dtype=torch.int32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        while True:
            for i in range(check_every):
                check(lib.sr_uv_chart_hook(_p(adj), _p(label), F, _p(cid), _p(changed), _stream()), "uv_chart_hook")
                flags[i:i + 1].copy_(changed)
            if not bool(flags[-1]):
                return cid


def uv_chart_project(verts, chart_off, uv_vert, chart_label):
    """-> (uvl [T,2] float64 chart-local coordinates, box [C,2] float64 chart extents) of the UV vertices uv_vert [T]
    grouped by chart (chart_off [C+1]), projected along the directions chart_label [C] int32."""
    _need_cuda(verts, chart_off, uv_vert, chart_label)
    C, T, dev = chart_label.shape[0], uv_vert.shape[0], verts.device
    uvl = torch.empty((T, 2), dtype=torch.float64, device=dev)
    box = torch.empty((C, 2), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().sr_uv_chart_project(_p(verts), C, _p(chart_off), _p(uv_vert), _p(chart_label), _p(uvl),
                                              _p(box), _stream()), "uv_chart_project")
    return uvl, box


def uv_place(uvl, uv_chart, offset, scale):
    """-> vt [T,2] float32 = offset[uv_chart] + scale * uvl."""
    _need_cuda(uvl, uv_chart, offset)
    T = uvl.shape[0]
    vt = torch.empty((T, 2), dtype=torch.float32, device=uvl.device)
    with torch.cuda.device(uvl.device):
        check(_lib.load().sr_uv_place(_p(uvl), _p(uv_chart), T, _p(offset), float(scale), _p(vt), _stream()),
              "uv_place")
    return vt


def uv_coverage(vt, ft, R, want_bad=True):
    """-> (count [R,R] int32 UV faces per texel centre, bad [F] uint8 faces on a texel counted twice, or None)."""
    _need_cuda(vt, ft)
    F, dev = ft.shape[0], vt.device
    count = torch.empty((R, R), dtype=torch.int32, device=dev)
    bad = torch.empty(F, dtype=torch.uint8, device=dev) if want_bad else None
    with torch.cuda.device(dev):
        check(_lib.load().sr_uv_coverage(_p(vt), _p(ft), F, int(R), _p(count), _p(bad), _stream()), "uv_coverage")
    return count, bad


TEXTURE_MAX_SLOTS = 64     # SR_TEXTURE_MAX_SLOTS


def texture_accumulate(texel_face, texel_bary, verts_screen, faces, vert_weight, face_usable, image, frame_id, slots):
    """One frame into the texture slots (csrc/texture_bake.cu).  texel_face [T] int32, texel_bary [T,3] of the covered
    atlas texels; verts_screen [V,3] (col, row, Z); faces [F,3] int64; vert_weight [V]; face_usable [F] uint8; image
    [H,W,3] uint8; slots = dict(rgb [S,3,T], alpha [S,T], view [S,T] int32, min_alpha [T], min_slot [T] int32),
    updated in place."""
    _need_cuda(texel_face, texel_bary, verts_screen, faces, vert_weight, face_usable, image)
    S, T = slots["alpha"].shape
    V, F = verts_screen.shape[0], faces.shape[0]
    H, W = image.shape[0], image.shape[1]
    if image.dim() != 3 or image.shape[2] != 3 or image.dtype != torch.uint8:
        raise ValueError("texture_accumulate: image must be [H,W,3] uint8")
    if texel_face.numel() != T or texel_bary.numel() != 3 * T or vert_weight.numel() != V or face_usable.numel() != F:
        raise ValueError("texture_accumulate: inconsistent shapes")
    with torch.cuda.device(image.device):
        check(_lib.load().sr_texture_accumulate(
            T, S, _p(texel_face), _p(texel_bary), _p(verts_screen), _p(faces), V, F, _p(vert_weight), _p(face_usable),
            _p(image), int(H), int(W), int(frame_id), _p(slots["rgb"]), _p(slots["alpha"]), _p(slots["view"]),
            _p(slots["min_alpha"]), _p(slots["min_slot"]), _stream()), "texture_accumulate")


def texture_finish(texel_index, slots, c0, min_views, n_texels):
    """count / mask_final / view_id / per-channel median of the filled slots at the covered texels texel_index [T]
    int64 of an atlas of n_texels -> (tex_median [n,3] float32, mask_final [n] uint8, view_id [n] int32, count [n]
    int32); texels outside texel_index get 0 / 0 / -1 / 0."""
    _need_cuda(texel_index)
    S, T = slots["alpha"].shape
    dev = texel_index.device
    med = torch.zeros((n_texels, 3), dtype=torch.float32, device=dev)
    mask = torch.zeros(n_texels, dtype=torch.uint8, device=dev)
    view = torch.full((n_texels,), -1, dtype=torch.int32, device=dev)
    count = torch.zeros(n_texels, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().sr_texture_finish(T, S, _p(texel_index), _p(slots["rgb"]), _p(slots["alpha"]),
                                            _p(slots["view"]), float(c0), int(min_views), _p(med), _p(mask), _p(view),
                                            _p(count), _stream()), "texture_finish")
    return med, mask, view, count


def mip_levels(Ht, Wt):
    """Level table of sr_texture_mips' pyramid for an Ht x Wt atlas: int64 [L,3] rows (first texel, H_l, W_l), with
    W_{l+1} = ceil(W_l / 2), H_{l+1} = ceil(H_l / 2) down to 1x1 (host tensor)."""
    Ht, Wt = int(Ht), int(Wt)
    if Ht <= 0 or Wt <= 0:
        raise ValueError("mip_levels: the atlas must not be empty, got %d x %d" % (Ht, Wt))
    rows, off = [(0, Ht, Wt)], Ht * Wt
    while Ht > 1 or Wt > 1:
        Ht, Wt = (Ht + 1) // 2, (Wt + 1) // 2
        rows.append((off, Ht, Wt))
        off += Ht * Wt
    return torch.tensor(rows, dtype=torch.int64)


def texture_mips(texture_u8, coverage):
    """Coverage-weighted mip pyramid of an atlas (csrc/avatar_texture.cu).  texture_u8 [Ht,Wt,3] uint8 in its own
    channel order, coverage [Ht,Wt] (bool or uint8, nonzero = covered) -> (mips [texels,4] float32 = (r, g, b, w) of
    every level, levels = mip_levels(Ht, Wt))."""
    _need_cuda(texture_u8, coverage)
    if texture_u8.dim() != 3 or texture_u8.shape[2] != 3 or texture_u8.dtype != torch.uint8:
        raise ValueError("texture_mips: the atlas must be [Ht,Wt,3] uint8, got %s %s"
                         % (tuple(texture_u8.shape), texture_u8.dtype))
    Ht, Wt = texture_u8.shape[0], texture_u8.shape[1]
    if tuple(coverage.shape) != (Ht, Wt) or coverage.dtype not in (torch.bool, torch.uint8):
        raise ValueError("texture_mips: coverage must be [Ht,Wt] = [%d,%d] bool or uint8" % (Ht, Wt))
    levels = mip_levels(Ht, Wt)
    n = int(levels[-1, 0] + levels[-1, 1] * levels[-1, 2])
    tex = texture_u8.contiguous()
    cov = coverage.to(torch.uint8).contiguous()
    mips = torch.empty((n, 4), dtype=torch.float32, device=tex.device)
    with torch.cuda.device(tex.device):
        check(_lib.load().sr_texture_mips(_p(tex), _p(cov), int(Ht), int(Wt), _p(mips), _stream()), "texture_mips")
    global LAUNCHES
    LAUNCHES += levels.shape[0] - 1        # one launch per level
    return mips, levels


def shade_textured(pix_to_face, bary, verts_screen, faces, ft, vt, mips, levels, background=(1., 1., 1.)):
    """Unlit trilinear-filtered atlas lookup on rasteriser fragments (csrc/avatar_texture.cu).  pix_to_face
    [N,H,W(,1)] packed ids n*F + f, bary [N,H,W(,1),3], verts_screen [N,V,3] (col, row, Z), faces / ft [F,3], vt [T,2],
    (mips, levels) of texture_mips; background = 3 floats or a uint8 image [N,H,W,3] in the atlas' channel order ->
    images [N,H,W,4]: (rgb, 1) on covered pixels, (background, 0) elsewhere."""
    bg_img = background if torch.is_tensor(background) else None
    _need_cuda(pix_to_face, bary, verts_screen, faces, ft, vt, mips, bg_img)
    vs = verts_screen.detach().contiguous().float()
    if vs.dim() != 3 or vs.shape[2] != 3:
        raise ValueError("shade_textured: verts_screen must be [N,V,3]")
    N, V, _ = vs.shape
    if pix_to_face.dim() not in (3, 4) or pix_to_face.shape[0] != N:
        raise ValueError("shade_textured: pix_to_face must be [N,H,W] or [N,H,W,1] with N = %d" % N)
    H, W = int(pix_to_face.shape[1]), int(pix_to_face.shape[2])
    p2f = pix_to_face.contiguous().to(torch.int64)
    br = bary.detach().contiguous().float()
    fc = faces.contiguous().to(torch.int64)
    ftc = ft.contiguous().to(torch.int64)
    vtc = vt.detach().contiguous().float()
    if p2f.numel() != N * H * W or br.numel() != 3 * N * H * W:
        raise ValueError("shade_textured: pix_to_face / bary do not match [N,H,W] = [%d,%d,%d]" % (N, H, W))
    if fc.dim() != 2 or fc.shape[1] != 3 or ftc.shape != fc.shape or vtc.dim() != 2 or vtc.shape[1] != 2:
        raise ValueError("shade_textured: faces and ft must be [F,3] and vt [T,2]")
    Ht, Wt = int(levels[0, 1]), int(levels[0, 2])
    n = int(levels[-1, 0] + levels[-1, 1] * levels[-1, 2])
    mips = mips.contiguous()
    if mips.dtype != torch.float32 or tuple(mips.shape) != (n, 4):
        raise ValueError("shade_textured: mips must be the [%d,4] float32 pyramid of the level table" % n)
    col = None
    if bg_img is not None:
        if bg_img.dtype != torch.uint8 or tuple(bg_img.shape) != (N, H, W, 3):
            raise ValueError("shade_textured: a background image must be [N,H,W,3] = [%d,%d,%d,3] uint8" % (N, H, W))
        bg_img = bg_img.contiguous()
    else:
        col = (C.c_float * 3)(*[float(c) for c in background])
    out = torch.empty((N, H, W, 4), dtype=torch.float32, device=vs.device)
    with torch.cuda.device(vs.device):
        check(_lib.load().sr_shade_textured(_p(p2f), _p(br), N, H, W, _p(vs), V, _p(fc), _p(ftc), fc.shape[0], _p(vtc),
                                            vtc.shape[0], _p(mips), Ht, Wt, _p(bg_img), col, _p(out),
                                            _stream()), "shade_textured")
    return out


_KERNELS_PER_CALL["shade_textured"] = 1


LBSW_MAX_K = 32           # SR_LBSW_MAX_K
LBSW_MAX_C = 32           # SR_LBSW_MAX_C


def lbsw_field(bmins, bmaxs, resolutions, verts, vert_ws, align_corners=False, k=5, want_centres=False):
    """Inverse-distance blend of the skin weights of the k nearest vertices at every voxel centre (csrc/lbsw_field.cu):
    verts [V,3], vert_ws [V,C] float32 CUDA, (W,H,D) = resolutions -> field [1,C,D,H,W] (and the voxel centres
    [W*H*D,3], x fastest, with want_centres).  The centres are bit-identical to utils.LBSWsmpl.voxel_centres."""
    _need_cuda(verts, vert_ws)
    if verts.dtype != torch.float32 or vert_ws.dtype != torch.float32:
        raise ValueError("lbsw_field: verts and vert_ws must be float32")
    verts = verts.reshape(-1, 3).contiguous()
    V, Cc = verts.shape[0], vert_ws.shape[-1]
    vert_ws = vert_ws.reshape(V, Cc).contiguous()
    W, H, D = [int(r) for r in resolutions]
    lo = (C.c_float * 3)(*torch.as_tensor(bmins, dtype=torch.float32).reshape(3).tolist())
    hi = (C.c_float * 3)(*torch.as_tensor(bmaxs, dtype=torch.float32).reshape(3).tolist())
    field = torch.empty((1, Cc, D, H, W), dtype=torch.float32, device=verts.device)
    centres = torch.empty((W * H * D, 3), dtype=torch.float32, device=verts.device) if want_centres else None
    with torch.cuda.device(verts.device):
        check(_lib.load().sr_lbsw_knn_blend(_p(verts), _p(vert_ws), V, Cc, lo, hi, W, H, D, int(bool(align_corners)),
                                            int(k), _p(field), _p(centres), _stream()), "lbsw_knn_blend")
    return (field, centres) if want_centres else field


def lbsw_smooth(field, times, cut=0.0):
    """`times` Jacobi passes of the damped 6-neighbour smoother with per-voxel renormalisation over field [1,C,D,H,W]
    float32 CUDA (two buffers in ping-pong, one launch per pass); with cut > 0, values below it become 0 after the last
    pass (after the blend itself when times == 0).  Returns a new volume; `field` is not modified."""
    _need_cuda(field)
    if field.dtype != torch.float32 or field.dim() != 5 or field.shape[0] != 1:
        raise ValueError("lbsw_smooth: field must be [1,C,D,H,W] float32")
    _, Cc, D, H, W = field.shape
    lib = _lib.load()
    src = field.contiguous()
    with torch.cuda.device(field.device):
        if times <= 0:
            src = src.clone()
            if cut > 0:
                check(lib.sr_lbsw_cut(_p(src), src.numel(), float(cut), _stream()), "lbsw_cut")
            return src
        bufs = [torch.empty_like(src), torch.empty_like(src) if times > 1 else None]
        for t in range(times):
            dst = bufs[t % 2]
            check(lib.sr_lbsw_smooth_pass(_p(src), _p(dst), Cc, D, H, W, float(cut) if t == times - 1 else 0.0,
                                          _stream()), "lbsw_smooth_pass")
            src = dst
    return src


def frames_decode(img_store, mask_store, normal_store, frame_ids, W, outputs=("img", "mask", "normal")):
    """One training batch from the device frame store (csrc/frames.cu): img_store / normal_store uint8 [F,H,W,3] in
    file order (normal_store may be None), mask_store int32 [F,H,ceil(W/32)] bit-packed, frame_ids host int64 [N] (a
    list or CPU tensor) -> {'img' [N,H,W,3], 'mask' [N,H,W], 'normal' [N,H,W,3]} fp32 on the store's device, for the
    names in `outputs`, bit-identical to SceneDataset.__getitem__.  ValueError for an id outside [0, F)."""
    _need_cuda(img_store, mask_store, normal_store)
    F, H = int(mask_store.shape[0]), int(mask_store.shape[1])
    ids = torch.as_tensor(frame_ids, dtype=torch.int64).reshape(-1)
    if ids.is_cuda:
        raise ValueError("frames_decode: frame ids are host integers (checked before the launch)")
    if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= F):
        raise ValueError("frames_decode: frame id out of range [0, %d): %s" % (F, ids.tolist()))
    N, dev = ids.numel(), mask_store.device
    shapes = {"img": (N, H, W, 3), "mask": (N, H, W), "normal": (N, H, W, 3)}
    outs = {k: torch.empty(shapes[k], dtype=torch.float32, device=dev) for k in outputs}
    with torch.cuda.device(dev):
        dids = ids.to(dev)
        check(_lib.load().sr_frames_decode(_p(img_store), _p(mask_store), _p(normal_store), F, H, int(W),
                                           _p(dids), N, _p(outs.get("img")), _p(outs.get("mask")),
                                           _p(outs.get("normal")), _stream()), "frames_decode")
    return outs


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


def _gs_shape(inp, grid, *others):
    """(N, C, D, H, W, P) after the checks the kernels rely on: a 5-D volume, a [N,Do,Ho,Wo,3] grid with the
    volume's batch size, and every tensor on the volume's device in its dtype (the kernel reads each through a
    pointer of that type)."""
    _need_cuda(inp, grid, *others)
    if inp.dim() != 5 or grid.dim() != 5 or grid.shape[-1] != 3:
        raise RuntimeError("grid_sampler_3d: expected a volume [N,C,D,H,W] and a grid [N,Do,Ho,Wo,3], got %s and %s"
                           % (tuple(inp.shape), tuple(grid.shape)))
    if grid.shape[0] != inp.shape[0]:
        raise RuntimeError("grid_sampler_3d: volume and grid have batch sizes %d and %d"
                           % (inp.shape[0], grid.shape[0]))
    for t in (grid,) + others:
        if t.dtype != inp.dtype or t.device != inp.device:
            raise RuntimeError("grid_sampler_3d: expected %s tensors on %s like the volume, got %s on %s"
                               % (inp.dtype, inp.device, t.dtype, t.device))
    N, Cc, D, H, W = inp.shape
    return N, Cc, D, H, W, grid.shape[1] * grid.shape[2] * grid.shape[3]


def grid_sample3d_forward(inp, grid, want_corner_idx=False):
    N, Cc, D, H, W, P = _gs_shape(inp, grid)
    Do, Ho, Wo = grid.shape[1:4]
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
    N, Cc, D, H, W, P = _gs_shape(inp, grid, grad_output)
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
    N, Cc, D, H, W, P = _gs_shape(inp, grid, grad_output, gg_input, gg_grid)
    if gg_input.shape != inp.shape:
        raise RuntimeError("grid_sampler_3d: gg_input has shape %s, the volume %s"
                           % (tuple(gg_input.shape), tuple(inp.shape)))
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
        (e.g. the SDF value without the 256-d feature): same buffers, narrower npad.  One view per n_out: later calls
        return it again, so its copies and tensor-core packs exist (and are refreshed on refold) once."""
        for c in self._children:
            if c.desc.layer[c.desc.n_layers - 1].n == n_out:
                return c
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
        # short lists: one column-split launch per layer instead of the persistent engine's per-tile latency;
        # the list is longer than SMALL_CAP only in degenerate cases -- then the persistent engine takes the rest
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
    device->host read happens once per tensor value, not once per trace.  Each entry holds its tensor, so
    no other tensor can be allocated at a cached address and hit a stale entry."""
    if not t.is_cuda:
        return tuple(float(x) for x in t.detach().reshape(-1).tolist())
    key = (t.device.index, t.data_ptr(), t._version, t.numel())
    hit = _host_cache.get(key)
    if hit is None:
        if len(_host_cache) > 64:
            _host_cache.clear()
        hit = (t, tuple(float(x) for x in t.detach().reshape(-1).tolist()))
        _host_cache[key] = hit
    return hit[1]


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
    _need_cuda(rays, init_pts)
    dev = init_pts.device
    P = init_pts.shape[0]
    if P == 0:
        pts, conv = init_pts.detach().float().clone(), torch.zeros((0,), dtype=torch.bool, device=dev)
        return (pts, conv, torch.zeros((times + 3,), dtype=torch.int32, device=dev)) if return_counters \
            else (pts, conv)
    tp = TraceParams()
    tp.cam_pos[:] = _host_floats(cam_pos)[:3]
    tp.dthreshold, tp.athreshold, tp.w1, tp.w2 = float(dthreshold), float(athreshold), float(w1), float(w2)
    if mode == "auto":
        mode = "tc" if (TC_ENABLED and P >= TC_MIN_POINTS) else "reverse"
    if mode == "tc":
        return _trace_surface_points_tc(sdf_net, def_net, lbs, tp, rays, init_pts, batch_inds, conds, times,
                                        return_counters)
    pts = init_pts.detach().contiguous().float().clone()
    rays = rays.detach().contiguous().float()
    bi = batch_inds.contiguous().to(torch.int64) if batch_inds is not None else None
    conds = conds.detach().contiguous().float() if conds is not None else None
    condlen = conds.shape[-1] if conds is not None else 0
    conv = torch.zeros((P,), dtype=torch.bool, device=dev)
    lists = [torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(2)]
    counters = torch.zeros((times + 3,), dtype=torch.int32, device=dev)
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
        self._wb_head = {}     # n_keep -> pack of the first n_keep rows of the input layer's W^T (wb_head)
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
            for n_keep, buf in self._wb_head.items():
                self._pack_head(n_keep, buf)

    def _pack_head(self, n_keep, buf):
        L = self.layers[0]
        e = L["_e"]
        check(_lib.load().sr_tc_pack_weights(_p(e["wt"]), n_keep, L["n"], e["wt"].shape[1], _p(buf), _stream()),
              "tc_pack_weights")

    def wb_head(self, n_keep):
        """Reverse-sweep operand of the input layer restricted to its first n_keep inputs (a narrow launch when
        n_keep <= 64), for sweeps that need only those columns of the input gradient: the tracer's translator keeps the
        positional-encoding part, not the latent code's.  Packed on first use, refreshed by repack()."""
        buf = self._wb_head.get(n_keep)
        if buf is None:
            lib = _lib.load()
            buf = torch.empty((lib.sr_tc_weight_bytes(n_keep, self.layers[0]["n"]),), dtype=torch.uint8,
                              device=self.fused.device)
            with torch.cuda.device(self.fused.device):
                self._pack_head(n_keep, buf)
            self._wb_head[n_keep] = buf
        return buf


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


def _tc_mlp_backward(lib, tcn, cot, bufs, acts, P, m_dev, g_out, g_skip, n_keep):
    """Cotangent rows `cot` [P][>= n_last] of the net outputs -> d/d(embedded input) in g_out (first n_keep columns),
    the skip layer's part in g_skip.  acts = the forward sweep's tiles; bufs = a pair of staging tile buffers the layers
    alternate between; m_dev: optional device-side row count."""
    global LAUNCHES
    L = len(tcn.layers)
    acts_c = (C.c_void_p * max(L - 1, 1))(*[a.data_ptr() for a in acts])
    head = tcn.wb_head(n_keep) if n_keep < tcn.layers[0]["k"] else None
    rc = lib.sr_tc_mlp_backward(tcn.c_layers, L, P, g_out.shape[1], tcn.fused.desc.d_in, 1, _p(cot), cot.shape[1],
                                None, acts_c, None, _p(bufs[0]), _p(bufs[1]), None, None, 0, None, None, _p(g_out),
                                _p(g_skip), g_skip.shape[1], _p(head), n_keep, 0, _p(m_dev), _stream())
    if rc == _lib.SR_EUNSUPPORTED:
        raise RuntimeError("selfrecon_b200: the tensor-core reverse sweep takes at most one skip layer; "
                           "use the fp32 engine (trace mode 'reverse', shade_geometry) for this network")
    check(rc, "tc_mlp_backward")
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
        self.side_stream = torch.cuda.Stream(device=dev)
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
                                  _p(B.cot_d) if def_net is not None else None, 32, _p(B.aux), _stream()),
              "tc_trace_mid")
        if a_out is None:
            break
        # ---- reverse sweeps + update
        if dual:
            side.wait_stream(main)
            with torch.cuda.stream(side):
                _tc_mlp_backward(lib, td, B.cot_d, B.A_d, B.acts_d, P, m_dev, B.gd, B.gskip_d, 3 + 6 * dd.multires)
        _tc_mlp_backward(lib, ts, B.cot_s, B.A, B.acts_s, P, m_dev, B.gs, B.gskip, ds.d_in)
        if dual:
            main.wait_stream(side)
        elif def_net is not None:
            _tc_mlp_backward(lib, td, B.cot_d, B.A, B.acts_d, P, m_dev, B.gd, B.gskip, 3 + 6 * dd.multires)
        has_skip = any(l["skip"] for l in ts.layers)
        check(lib.sr_tc_trace_update(_p(idx), _p(m_dev), P, _p(pts), _p(B.gs), B.gs.shape[1],
                                     _p(B.gskip) if has_skip else None, B.gskip.shape[1],
                                     _p(B.gd) if def_net is not None else None,
                                     B.gd.shape[1] if def_net is not None else 0, _p(B.aux), ds.multires,
                                     pw_s, dd.multires if dd is not None else 0, pw_d, _p(a_out),
                                     _p(counters[it + 1:it + 2]), _stream()),
              "tc_trace_update")


def _trace_surface_points_tc(sdf_net, def_net, lbs, tp, rays, init_pts, batch_inds, conds, times, return_counters):
    """trace_surface_points with the dense layers on the tensor-core engine (reverse-mode sweeps), for
    P > 0 rays.  A trace is ~35 launches per iteration, all with static shapes and device-side counts, so
    from the second call with the same configuration (ray count, networks, thresholds, PE weights) the
    whole trace is replayed as one CUDA graph (SELFRECON_B200_GRAPHS=0 keeps it eager)."""
    global LAUNCHES
    dev = init_pts.device
    P = init_pts.shape[0]
    lib = _lib.load()
    condlen = conds.shape[-1] if conds is not None else 0
    n_frames = lbs.A.shape[0] if lbs is not None else (conds.shape[0] if conds is not None else 1)
    ds, dd = sdf_net.desc, (def_net.desc if def_net is not None else None)
    # buffers depend on shapes only; the captured graph also on everything a launch bakes in
    key = (dev.index, P, tuple(ds.layer[i].n for i in range(ds.n_layers)),
           tuple(dd.layer[i].n for i in range(dd.n_layers)) if dd is not None else (), n_frames, condlen,
           conds.shape[0] if conds is not None else 0, times)
    sig = (sdf_net.uid, def_net.uid if def_net is not None else -1,
           lbs.ws_cl.data_ptr() if lbs is not None else 0, tuple(tp.cam_pos), tp.dthreshold, tp.athreshold,
           tp.w1, tp.w2, tuple(ds.pe_w[i] for i in range(ds.multires)),
           tuple(dd.pe_w[i] for i in range(dd.multires)) if dd is not None else (), TC_DUAL_STREAM)
    G = _tc_trace_ctx.get(key)
    if G is None:
        if len(_tc_trace_ctx) >= 4:
            _tc_trace_ctx.pop(next(iter(_tc_trace_ctx)))
        G = _TcTraceCtx(dev, P, sdf_net, def_net, n_frames, condlen, times)
        _tc_trace_ctx[key] = G
    if G.sig != sig:          # new weights / thresholds: the old graph is stale, buffers are not
        G.sig, G.graph, G.calls = sig, None, 0
    ts, td = tc_net(sdf_net), (tc_net(def_net) if def_net is not None else None)
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


class _TcShadeBuffers:
    """Work buffers of the SDF's reverse-mode gradient in shade_and_render_tc for up to `cap` points (the kept
    activation tiles alone take ~0.9 GB at 50 000 points)."""

    def __init__(self, dev, cap, sdf_full):
        lib = _lib.load()
        d = sdf_full.desc
        f32 = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)   # noqa: E731
        u8 = lambda n: torch.empty((n,), dtype=torch.uint8, device=dev)           # noqa: E731
        self.cap = cap
        self.ld = _pad(d.d_in, 32)
        self.emb = f32(cap, self.ld)
        self.A_in = u8(lib.sr_tc_act_bytes(cap, self.ld))
        self.acts = [u8(lib.sr_tc_act_bytes(cap, _pad(d.layer[i + 1].k, 32))) for i in range(d.n_layers - 1)]
        self.out = f32(cap, d.layer[d.n_layers - 1].n)          # f + features
        widest = max([32] + [_pad(d.layer[l].n, 32) for l in range(d.n_layers - 1)])
        self.A = [u8(lib.sr_tc_act_bytes(cap, widest)) for _ in range(2)]
        self.cot = torch.zeros((cap, 32), dtype=torch.float32, device=dev)
        self.cot[:, 0] = 1.0                                     # d f / d f: the reverse sweep's seed
        self.g_out = f32(cap, self.ld)
        self.g_skip = f32(cap, self.ld)
        self.grad = f32(cap, 3)


# one buffer set per (device, SDF layer shapes), grown (by at least a quarter, in steps of 4096 points) when a call
# brings more points than it holds: a point count that changes from frame to frame keeps hitting it
_tc_shade_bufs = {}


def _tc_shade_key(dev, d):
    """The buffer set's key: every size _TcShadeBuffers reads from the descriptor.  The activation tiles are sized by
    each layer's input width k, which the output widths n and d_in do not fix (a skip layer's k is n + d_in)."""
    return (dev.index, tuple((d.layer[i].n, d.layer[i].k) for i in range(d.n_layers)), d.d_in)


def _sdf_grad_tc(lib, sdf_full, pts, P):
    """SDF value + features and grad f in reverse mode: one value-only forward sweep keeping its activation tiles, one
    reverse sweep from a cotangent of 1 on f (the value-only view's layers: the last one is 1 wide), then the chain
    through the positional encoding.  Returns views of the cached buffers: out [P, 1 + nfeat], grad [P, 3] and the
    encoding's cotangent without the skip layer's part, g_out [P, pad32(d_in)]."""
    dev = pts.device
    d = sdf_full.desc
    key = _tc_shade_key(dev, d)
    B = _tc_shade_bufs.get(key)
    if B is None or B.cap < P:
        cap = _pad(max(P, B.cap + B.cap // 4 if B is not None else 0), 4096)
        _tc_shade_bufs.pop(key, None)
        B = None                                         # drop the smaller set before allocating its successor
        B = _tc_shade_bufs[key] = _TcShadeBuffers(dev, cap, sdf_full)
    ts, tv = tc_net(sdf_full), tc_net(sdf_full.truncated_last(1))
    pw = (C.c_float * 16)(*[d.pe_w[i] for i in range(16)])
    emb, out, grad, g_out = B.emb[:P], B.out[:P], B.grad[:P], B.g_out[:P]
    check(lib.sr_tc_embed(_p(pts), P, d.multires, pw, 1, None, None, 0, 0, _p(emb), B.ld, None, None, _stream()),
          "tc_embed")
    _tc_mlp(lib, ts, emb, 1, out, B.A_in, B.acts)
    _tc_mlp_backward(lib, tv, B.cot, B.A, B.acts, P, None, g_out, B.g_skip, d.d_in)
    has_skip = any(l["skip"] for l in ts.layers)
    check(lib.sr_tc_embed_backward(_p(pts), P, d.multires, pw, 1, _p(g_out), B.ld, _p(B.g_skip) if has_skip else None,
                                   B.ld, _p(grad), _stream()), "tc_embed_backward")
    return out, grad, g_out


def shade_and_render_tc(sdf_full, def_net, lbs, render_net, pts, rays, batch_inds, conds, nfeat=256,
                        deformed_normals=False, cam_R0=None):
    """Shading of the infer path on the tensor-core engine: grad f of the SDF in reverse mode (one value-only forward
    sweep + one reverse sweep), the translator's sweep with forward tangents (4 rows per point: its 3x3 Jacobian),
    pointwise geometry, then the rendering network.
    Returns (normals, cardinal rays, rgb, D(p), inverse-ok mask); with `deformed_normals` also the deformed-surface
    normal normalize(J^-T grad f) [P,3] from the same pointwise pass, rotated into the debug image's frame
    diag(-1,1,-1) cam_R0^T n when a 3x3 `cam_R0` is given."""
    _need_cuda(pts, rays)
    dev = pts.device
    P = pts.shape[0]
    pts = pts.detach().contiguous().float()
    rays = rays.detach().contiguous().float()
    bi = batch_inds.contiguous().to(torch.int64) if batch_inds is not None else None
    if P == 0:
        # an empty ray set (trace_surface_points returns empty tensors for one): the kernels refuse P = 0
        rd = render_net.desc
        e3 = lambda: torch.empty((0, 3), dtype=torch.float32, device=dev)   # noqa: E731
        out = (e3(), e3(), torch.empty((0, rd.layer[rd.n_layers - 1].n), dtype=torch.float32, device=dev), e3(),
               torch.empty((0,), dtype=torch.bool, device=dev))
        return out + (e3(),) if deformed_normals else out
    lib = _lib.load()
    with torch.cuda.device(dev):
        if TC_DUAL_STREAM and def_net is not None:
            # SDF and translator sweeps are independent: second stream (see _tc_trace_body)
            main = torch.cuda.current_stream()
            side = _side_stream(dev)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                o4 = tc_mlp_forward(def_net, pts, ch=4, conds=conds, batch_inds=bi)
            f_feat, grad, _ = _sdf_grad_tc(lib, sdf_full, pts, P)
            main.wait_stream(side)
            o4.record_stream(main)
        else:
            f_feat, grad, _ = _sdf_grad_tc(lib, sdf_full, pts, P)
            o4 = tc_mlp_forward(def_net, pts, ch=4, conds=conds, batch_inds=bi) if def_net is not None else None
        normals = torch.empty((P, 3), dtype=torch.float32, device=dev)
        crays = torch.empty((P, 3), dtype=torch.float32, device=dev)
        dpos = torch.empty((P, 3), dtype=torch.float32, device=dev)
        ok = torch.empty((P,), dtype=torch.bool, device=dev)
        if deformed_normals:
            defn = torch.empty((P, 3), dtype=torch.float32, device=dev)
            R0 = None
            if cam_R0 is not None:
                R0 = (C.c_float * 9)(*[float(x) for x in cam_R0.detach().reshape(9).float().cpu().tolist()])
            check(lib.sr_tc_shade_point_deformed(P, _p(pts), _p(rays), _p(bi), _p(grad), _p(o4), _lbs_ref(lbs),
                                                 _p(normals), _p(crays), _p(dpos), _p(ok), _p(defn), R0, _stream()),
                  "tc_shade_point_deformed")
        else:
            check(lib.sr_tc_shade_point(P, _p(pts), _p(rays), _p(bi), _p(grad), _p(o4), _lbs_ref(lbs),
                                        _p(normals), _p(crays), _p(dpos), _p(ok), _stream()), "tc_shade_point")
        rd = render_net.desc
        ld = _pad(rd.d_in, 32)
        emb = torch.empty((P, ld), dtype=torch.float32, device=dev)
        pw = (C.c_float * 16)(*[rd.pe_w[i] for i in range(16)])
        check(lib.sr_tc_render_embed(P, _p(pts), _p(crays), _p(normals), _p(f_feat), f_feat.shape[1], 1, nfeat, 1,
                                     rd.multires, pw, _p(emb), ld, _stream()), "tc_render_embed")
        rn = tc_net(render_net)
        rgb = torch.empty((P, rn.layers[-1]["n"]), dtype=torch.float32, device=dev)
        _tc_mlp(lib, rn, emb, 1, rgb)
    if deformed_normals:
        return normals, crays, rgb, dpos, ok, defn
    return normals, crays, rgb, dpos, ok


# ------------------------------------------------------------------------------------------------
# Front-normal network (csrc/normal_net.cu; generate_normals.py:116-166): convolutions as an implicit-im2col pack
# plus the tensor-core layer kernel, instance norm, and the map of the net output back onto the frame
# ------------------------------------------------------------------------------------------------
class TcConv:
    """One convolution on the tensor-core engine: weight [Cout, Cin, kh, kw] (Conv2d) or [Cin, Cout, kh, kw]
    (ConvTranspose2d, transposed=True) reordered once to [Cout, kh*kw*Cin] (tap-major, channel-minor) and packed;
    bias zero-padded to pad256(Cout).  pad_mode 'zeros' or 'reflect'; output_padding only for transposed."""

    def __init__(self, weight, bias, stride=1, pad=0, pad_mode="zeros", transposed=False, output_padding=0):
        _need_cuda(weight)
        w = weight.detach().float()
        if transposed:
            w = w.permute(1, 2, 3, 0)           # W[ci, co, ky, kx] -> [co, ky, kx, ci]
        else:
            w = w.permute(0, 2, 3, 1)           # W[co, ci, ky, kx] -> [co, ky, kx, ci]
        self.cout, self.kh, self.kw, self.cin = (int(s) for s in w.shape)
        self.K = self.kh * self.kw * self.cin
        self.W = tc_pack_weights(w.reshape(self.cout, self.K))
        self.bias = torch.zeros((_pad(self.cout, 256),), dtype=torch.float32, device=w.device)
        if bias is not None:
            self.bias[:self.cout] = bias.detach().float().reshape(-1)
        if pad_mode not in ("zeros", "reflect") or stride not in (1, 2):
            raise ValueError("TcConv: stride 1 or 2, pad_mode 'zeros' or 'reflect'")
        self.stride, self.pad, self.reflect = int(stride), int(pad), pad_mode == "reflect"
        self.transposed, self.output_padding = bool(transposed), int(output_padding)

    def out_size(self, H, W):
        if self.transposed:
            f = lambda n, k: (n - 1) * self.stride - 2 * self.pad + k + self.output_padding
        else:
            f = lambda n, k: (n + 2 * self.pad - k) // self.stride + 1
        return f(H, self.kh), f(W, self.kw)

    def row_bytes(self):
        return _lib.load().sr_tc_act_bytes(128, self.K) // 128


def conv2d(x, conv, workspace, act=_lib.SR_ACT_NONE, chunk_rows=None, out=None):
    """x fp32 channels-last [B,H,W,Cin] -> conv(x) fp32 [B,Ho,Wo,Cout] (act applied), through row chunks of the
    implicit im2col matrix packed into `workspace` (a uint8 CUDA buffer): each chunk is one sr_conv_pack and one
    sr_tc_linear.  chunk_rows (a multiple of 128) defaults to what the workspace holds."""
    _need_cuda(x, workspace)
    B, H, W, Cin = (int(s) for s in x.shape)
    if Cin != conv.cin or x.dtype != torch.float32 or not x.is_contiguous():
        raise ValueError("conv2d: expected contiguous fp32 [B,H,W,%d], got %s %s" % (conv.cin, x.dtype, tuple(x.shape)))
    Ho, Wo = conv.out_size(H, W)
    M = B * Ho * Wo
    cap = workspace.numel() // conv.row_bytes() // 128 * 128
    rows = cap if chunk_rows is None else int(chunk_rows)
    if rows < 128 or rows % 128 or rows > cap:
        raise ValueError("conv2d: chunks of %d rows (a multiple of 128, at most %d for this workspace)" % (rows, cap))
    if out is None:
        out = torch.empty((B, Ho, Wo, conv.cout), dtype=torch.float32, device=x.device)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        for r0 in range(0, M, rows):
            n = min(rows, M - r0)
            check(lib.sr_conv_pack(_p(x), B, H, W, Cin, conv.kh, conv.kw, conv.stride, conv.pad, int(conv.reflect),
                                   int(conv.transposed), Ho, Wo, r0, n, _p(workspace), _stream()), "conv_pack")
            dst = C.c_void_p(out.data_ptr() + r0 * conv.cout * 4)
            check(lib.sr_tc_linear(_p(workspace), _p(conv.W), _p(conv.bias), n, conv.cout, conv.K, conv.cout, int(act),
                                   1, None, 0, 1.0, None, 0, 0, dst, conv.cout, 0, conv.cout, None, None, 0, 0, 1.0,
                                   None, _stream()), "tc_linear")
    return out


def instance_norm_stats(y):
    """y fp32 [B,H,W,C] -> (mean, rstd) fp32 [B,C]: InstanceNorm2d's per-instance statistics (biased variance, eps
    1e-5), deterministic and independent of B."""
    _need_cuda(y)
    B, C_ = int(y.shape[0]), int(y.shape[-1])
    HW = y.numel() // (B * C_)
    lib = _lib.load()
    part = torch.empty((lib.sr_instance_norm_partial_bytes(B, HW, C_),), dtype=torch.uint8, device=y.device)
    mean = torch.empty((B, C_), dtype=torch.float32, device=y.device)
    rstd = torch.empty((B, C_), dtype=torch.float32, device=y.device)
    with torch.cuda.device(y.device):
        check(lib.sr_instance_norm_stats(_p(y), B, HW, C_, _p(part), _p(mean), _p(rstd), _stream()),
              "instance_norm_stats")
    return mean, rstd


def instance_norm_apply(y, mean, rstd, residual=None, relu=False, out=None):
    """out = relu?((y - mean) * rstd) (+ residual), all fp32 [B,H,W,C] (out may be y or residual)."""
    _need_cuda(y, mean, rstd, residual)
    B, C_ = int(y.shape[0]), int(y.shape[-1])
    if residual is not None and residual.shape != y.shape:
        raise ValueError("instance_norm_apply: residual %s, y %s" % (tuple(residual.shape), tuple(y.shape)))
    out = torch.empty_like(y) if out is None else out
    with torch.cuda.device(y.device):
        check(_lib.load().sr_instance_norm_apply(_p(y), B, y.numel() // (B * C_), C_, _p(mean), _p(rstd),
                                                 _p(residual), int(bool(relu)), _p(out), _stream()),
              "instance_norm_apply")
    return out


def normal_unwarp(net_out, boxes, fg, H, W):
    """net_out fp32 [B,S,S,3] (channels-last tanh output), boxes fp32 [B,4] (x, y, w, h), fg uint8 [B,H,W] (nonzero =
    foreground) or None -> uint8 BGR [B,H,W,3]: generate_normals.py:149-165 (grid_sample back onto the frame, zero
    where |n| < 1e-4 or background, (n*0.5 + 0.5)[::-1]*255 truncated)."""
    _need_cuda(net_out, boxes, fg)
    B, S = int(net_out.shape[0]), int(net_out.shape[1])
    if tuple(net_out.shape) != (B, S, S, 3) or tuple(boxes.shape) != (B, 4) or \
            (fg is not None and tuple(fg.shape) != (B, H, W)):
        raise ValueError("normal_unwarp: net_out [B,S,S,3], boxes [B,4], fg [B,H,W] expected")
    out = torch.empty((B, H, W, 3), dtype=torch.uint8, device=net_out.device)
    with torch.cuda.device(net_out.device):
        check(_lib.load().sr_normal_unwarp(_p(net_out.contiguous()), B, S, _p(boxes.float().contiguous()),
                                           _p(fg.contiguous() if fg is not None else None), int(H), int(W), _p(out),
                                           _stream()), "normal_unwarp")
    return out
