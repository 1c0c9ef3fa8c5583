"""Simplify and UV-unwrap the reconstructed template on the device, so texturing starts from tmp.ply:

    python -m selfreconcode_b200.uvmap --rec-root <result>      # <result>/tmp.ply -> <result>/template/uvmap.obj

then texture.bake_from_network(optNet, "<result>/template/uvmap.obj", out_dir) as before.  Steps (DESIGN.md section
3.3): read_mesh (PLY), simplify (parallel quadric edge collapse, csrc/mesh_simplify.cu), unwrap (26-direction charts,
orthographic projection, shelf packing, overlap check; csrc/uv_atlas.cu), write_obj."""
import argparse
import os
import os.path as osp
import sys

import numpy as np
import torch

from . import enable_dropin, ops

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}
_XYZ_TYPES = ("float", "float32", "double", "float64")
_COUNT_TYPES = ("uchar", "uint8", "int", "uint")
_INDEX_TYPES = ("int", "int32", "uint", "uint32")


def _parse_header(path, fh):
    if fh.readline().strip() != b"ply":
        raise ValueError("%s: not a PLY file" % path)
    fmt, elements = None, []
    while True:
        line = fh.readline()
        if not line:
            raise ValueError("%s: PLY header without end_header" % path)
        tok = line.decode("ascii", "replace").split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "end_header":
            break
        if tok[0] == "format" and len(tok) == 3:
            fmt = tok[1]
        elif tok[0] == "element" and len(tok) == 3:
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property" and elements and len(tok) == 3 and tok[1] in _PLY_TYPES:
            elements[-1][2].append((tok[2], tok[1]))
        elif tok[0] == "property" and elements and len(tok) == 5 and tok[1] == "list":
            elements[-1][2].append((tok[4], ("list", tok[2], tok[3])))
        else:
            raise ValueError("%s: unsupported PLY header line %r" % (path, line.strip()))
    if fmt not in ("ascii", "binary_little_endian"):
        raise ValueError("%s: unsupported PLY format %r (ascii or binary_little_endian)" % (path, fmt))
    names = [e[0] for e in elements]
    if names[:2] != ["vertex", "face"] or len(names) != 2:
        raise ValueError("%s: expected the elements vertex then face, got %s" % (path, names))
    vprops = elements[0][2]
    pos = {n: t for n, t in vprops}
    if any(isinstance(t, tuple) for _, t in vprops) or any(pos.get(c) not in _XYZ_TYPES for c in "xyz"):
        raise ValueError("%s: vertex x y z must be float or double scalars" % path)
    fprops = elements[1][2]
    if len(fprops) != 1 or not isinstance(fprops[0][1], tuple) or fprops[0][0] not in ("vertex_indices",
                                                                                          "vertex_index"):
        raise ValueError("%s: the face element must hold one vertex_indices list" % path)
    _, ct, it = fprops[0][1]
    if ct not in _COUNT_TYPES or it not in _INDEX_TYPES:
        raise ValueError("%s: unsupported face list types %s %s" % (path, ct, it))
    return fmt, elements[0][1], vprops, elements[1][1], ct, it


def _fan(counts, idx, path):
    """Polygons (counts [F], flat indices) -> triangles (0, i, i+1)."""
    if counts.size and counts.min() < 3:
        raise ValueError("%s: face with fewer than 3 vertices" % path)
    if counts.size and (counts == 3).all():
        return idx.reshape(-1, 3)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    tris = [np.stack([np.full(c - 2, idx[s]), idx[s + 1:s + c - 1], idx[s + 2:s + c]], 1) for s, c in zip(starts, counts)]
    return np.concatenate(tris, 0)


def read_mesh(path):
    """PLY (ascii or binary_little_endian) -> (V [V,3] float32, F [F,3] int64) host tensors.  Vertex x y z as float or
    double (other vertex properties skipped), one face list (count uchar / int / uint, index int / uint); a polygon
    becomes the fan (0, i, i+1).  Anything else is a ValueError naming the file."""
    with open(path, "rb") as fh:
        fmt, nv, vprops, nf, ct, it = _parse_header(path, fh)
        body = fh.read()
    names = [n for n, _ in vprops]
    try:
        if fmt == "ascii":
            tok = body.split()
            nvp = len(vprops)
            vals = np.array(tok[:nv * nvp], dtype=np.float64).reshape(nv, nvp)
            V = vals[:, [names.index(c) for c in "xyz"]]
            rest, counts, idx, k = tok[nv * nvp:], np.empty(nf, np.int64), [], 0
            for f in range(nf):
                c = int(rest[k])
                counts[f] = c
                idx.append(rest[k + 1:k + 1 + c])
                k += 1 + c
            idx = np.array([int(x) for row in idx for x in row], dtype=np.int64)
        else:
            vdt = np.dtype([(n, "<" + _PLY_TYPES[t]) for n, t in vprops])
            varr = np.frombuffer(body, dtype=vdt, count=nv)
            V = np.stack([varr[c].astype(np.float64) for c in "xyz"], 1)
            off = vdt.itemsize * nv
            cdt, idt = np.dtype("<" + _PLY_TYPES[ct]), np.dtype("<" + _PLY_TYPES[it])
            tri = np.dtype([("n", cdt), ("v", idt, (3,))])
            rows = np.frombuffer(body, dtype=tri, count=nf, offset=off) if len(body) >= off + tri.itemsize * nf \
                else None
            if rows is not None and (rows["n"] == 3).all():
                counts, idx = rows["n"].astype(np.int64), rows["v"].astype(np.int64).reshape(-1)
            else:
                counts, idx, k = np.empty(nf, np.int64), [], off
                for f in range(nf):
                    c = int(np.frombuffer(body, cdt, 1, k)[0])
                    counts[f] = c
                    idx.append(np.frombuffer(body, idt, c, k + cdt.itemsize).astype(np.int64))
                    k += cdt.itemsize + c * idt.itemsize
                idx = np.concatenate(idx) if idx else np.zeros(0, np.int64)
    except (IndexError, ValueError) as e:
        raise ValueError("%s: truncated or malformed PLY body (%s)" % (path, e))
    F = _fan(counts, idx, path) if nf else np.zeros((0, 3), np.int64)
    return torch.from_numpy(np.ascontiguousarray(V, dtype=np.float32)), torch.from_numpy(np.ascontiguousarray(F))


def write_obj(path, V, F, vt, ft):
    """`v`, `vt` and `f v/vt` (1-based) lines, numbers as %.9g so texture.load_obj_uv reads back the same float32s."""
    V, vt = [np.asarray(torch.as_tensor(x).cpu(), dtype=np.float32).astype(np.float64) for x in (V, vt)]
    F, ft = [np.asarray(torch.as_tensor(x).cpu(), dtype=np.int64) + 1 for x in (F, ft)]
    d = osp.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "w") as fh:
        fh.write("".join("v %.9g %.9g %.9g\n" % tuple(r) for r in V))
        fh.write("".join("vt %.9g %.9g\n" % tuple(r) for r in vt))
        fh.write("".join("f %d/%d %d/%d %d/%d\n" % (a, x, b, y, c, z) for (a, b, c), (x, y, z) in zip(F, ft)))


def _vertex_face_csr(F, nv):
    enable_dropin()
    from model.raster import vertex_face_csr
    return vertex_face_csr(F, nv)


def drop_broken(V, F):
    """Drops faces with a negative or out-of-range corner (marching cubes' -1), then vertices no face references.
    -> (V', F', dropped faces, dropped vertices)."""
    nv = V.shape[0]
    ok = ((F >= 0) & (F < nv)).all(1)
    F = F[ok]
    used = torch.zeros(nv, dtype=torch.bool, device=V.device)
    used[F.reshape(-1)] = True
    new_id = torch.cumsum(used.long(), 0) - 1
    df, dv = torch.stack([(~ok).sum(), (~used).sum()]).tolist()
    return V[used].contiguous(), new_id[F].contiguous(), df, dv


_NO_KEY = -1    # ~0 of the uint64 keys, as int64


def simplify_round(V, F, target):
    """One collapse round -> (V', F', number of collapses).  The edge table is mesh_reg's; the one readback is the
    number of selected edges, from which the new counts follow (each collapse removes one vertex and two faces)."""
    nv, nf = V.shape[0], F.shape[0]
    topo = ops.mesh_reg_topology(F, nv)
    csr = _vertex_face_csr(F, nv)
    Q, fixed = ops.simplify_quadrics(V, F, csr, topo)
    vstar, _, key = ops.simplify_edge_cost(V, F, csr, topo, Q, fixed)
    sel = ops.simplify_select(topo, key)
    n_sel = int(sel.sum())
    n = min(n_sel, (nf - target) // 2)
    if n <= 0:
        return V, F, 0
    if n < n_sel:   # last round: only the n lowest keys, so the face count lands on the target
        kth = torch.sort(torch.where(sel.bool(), key, torch.full_like(key, 2 ** 63 - 1))).values[n - 1]
        sel = (sel.bool() & (key <= kth)).to(torch.uint8)
    V, F = ops.simplify_collapse(V, F, topo.edges, sel, vstar, nv - n, nf - 2 * n)
    return V, F, n


def simplify(V, F, faces=30000, max_rounds=200):
    """Parallel quadric edge collapse of a CUDA mesh (V [V,3] float32, F [F,3] int64) down to `faces` faces ->
    (V', F', info).  info: faces_in, faces_out, rounds, faces_per_round, stop ('target', 'no valid collapse' or
    'max_rounds'), dropped_faces / dropped_vertices (broken corners and unreferenced vertices, dropped first)."""
    ops._need_cuda(V, F)
    target = int(faces)
    if target < 4:
        raise ValueError("simplify: faces must be at least 4, got %d" % target)
    V, F, df, dv = drop_broken(V.detach().contiguous().float(), F.detach().contiguous().long())
    if df or dv:
        print("[uvmap] dropped %d faces with a missing corner and %d unreferenced vertices" % (df, dv))
    info = dict(faces_in=F.shape[0], dropped_faces=df, dropped_vertices=dv, faces_per_round=[], rounds=0)
    if F.shape[0] == 0:
        raise ValueError("simplify: the mesh has no valid face")
    stop = "max_rounds"
    for r in range(int(max_rounds)):
        if F.shape[0] <= target + 1:
            stop = "target"
            break
        V, F, n = simplify_round(V, F, target)
        if n == 0:
            stop = "no valid collapse"
            break
        info["rounds"] = r + 1
        info["faces_per_round"].append(F.shape[0])
    else:
        if F.shape[0] <= target + 1:
            stop = "target"
    info.update(faces_out=F.shape[0], stop=stop)
    return V, F, info


def pack_charts(box, resolution, padding):
    """Shelf packing of chart boxes [C,2] (width >= height, any unit) into [0,1]^2 at one common scale -> (offsets
    [C,2] float64, scale).  Charts go in order of decreasing height (chart id on ties), left to right in rows whose
    height is their first chart's; every box keeps padding / resolution of gutter to its neighbours and to the atlas
    border.  The scale is the largest that fits, found by bisection."""
    box = np.asarray(box, dtype=np.float64).reshape(-1, 2)
    pad = float(padding) / float(resolution)
    order = np.lexsort((np.arange(box.shape[0]), -box[:, 1]))

    def place(s):
        offs = np.zeros_like(box)
        x, y, row = pad, pad, 0.0
        for c in order:
            w, h = box[c] * s
            if x + w + pad > 1.0 and x > pad:
                x, y, row = pad, y + row + pad, 0.0
            if x + w + pad > 1.0:
                return None
            offs[c] = (x, y)
            x += w + pad
            row = max(row, h)
        return offs if y + row + pad <= 1.0 else None

    hi = (1.0 - 2.0 * pad) / max(float(box.max()), 1e-30)
    lo, best = 0.0, place(hi)
    if best is not None:
        return best, hi
    for _ in range(64):
        mid = 0.5 * (lo + hi)
        o = place(mid)
        if o is None:
            hi = mid
        else:
            lo, best = mid, o
    if best is None:
        raise ValueError("pack_charts: %d charts do not fit with a %d-texel gutter at resolution %d"
                         % (box.shape[0], int(padding), int(resolution)))
    return best, lo


def _compact_ids(cid):
    """Chart ids (a representative face id per face) -> ids 0..C-1 in ascending representative order, and C."""
    F = cid.shape[0]
    root = torch.zeros(F, dtype=torch.int64, device=cid.device)
    root[cid] = 1
    cum = torch.cumsum(root, 0)
    return cum[cid] - 1, int(cum[-1])


class Atlas:
    """The charts of one unwrap: face_chart [F], chart_label [C], the (chart, vertex) UV vertices uv_chart / uv_vert
    [T], ft [F,3], chart-local uvl [T,2] and boxes [C,2]."""

    def __init__(self, V, F, face_chart, n_charts, label):
        nv, dev = V.shape[0], V.device
        self.face_chart, self.C = face_chart, n_charts
        self.chart_label = torch.zeros(n_charts, dtype=torch.int32, device=dev).scatter_(0, face_chart, label)
        keys, ft = torch.unique((face_chart[:, None] * nv + F).reshape(-1), sorted=True, return_inverse=True)
        self.uv_chart, self.uv_vert = keys // nv, keys % nv
        self.ft = ft.view(-1, 3)
        off = torch.searchsorted(self.uv_chart, torch.arange(n_charts + 1, dtype=torch.int64, device=dev))
        self.uvl, self.box = ops.uv_chart_project(V, off, self.uv_vert, self.chart_label)


def split_charts(atlas, bad):
    """Each chart holding a face flagged in bad [F] is cut in two at its median face centroid along its longer
    (chart-local u) axis: the first floor(n/2) faces by (centroid u, face id) against the rest.  -> new chart id per
    face (minimum face id of each part), compacted ascending, and the number of charts."""
    fc, dev = atlas.face_chart, bad.device
    F = fc.shape[0]
    flagged = torch.zeros(atlas.C, dtype=torch.bool, device=dev)
    flagged[fc[bad.bool()]] = True
    cu = atlas.uvl[:, 0][atlas.ft].mean(1)
    order = torch.argsort(cu, stable=True)
    order = order[torch.argsort(fc[order], stable=True)]
    counts = torch.bincount(fc, minlength=atlas.C)
    start = torch.cumsum(counts, 0) - counts
    rank = torch.empty(F, dtype=torch.int64, device=dev)
    rank[order] = torch.arange(F, device=dev) - start[fc[order]]
    part = (flagged[fc] & (rank >= counts[fc] // 2)).long()
    group = 2 * fc + part
    first = torch.full((2 * atlas.C,), F, dtype=torch.int64, device=dev)
    first.scatter_reduce_(0, group, torch.arange(F, device=dev), "amin")
    return _compact_ids(first[group])


def unwrap(V, F, resolution=1680, padding=4, max_angle=60., max_splits=64):
    """UV atlas of a CUDA mesh -> (vt [T,2] float32, ft [F,3] int64, info).  info: charts, scale, utilisation (covered
    texels / R^2), stretch_min / stretch_max (UV area / (scale^2 3-D area) over faces with area, from the fp64 chart coordinates), splits (overlap
    rounds), count (the coverage [R,R] int32)."""
    ops._need_cuda(V, F)
    R, pad = int(resolution), int(padding)
    if not (35. <= float(max_angle) <= 80.):
        raise ValueError("unwrap: max_angle must lie in [35, 80] degrees, got %r" % (max_angle,))
    if R <= 0 or pad < 1:
        raise ValueError("unwrap: resolution must be positive and padding at least 1 texel")
    V, F = V.detach().contiguous().float(), F.detach().contiguous().long()
    csr = _vertex_face_csr(F, V.shape[0])
    adj = ops.uv_face_adjacency(F, csr)
    _, area, label = ops.uv_labels(V, F, adj, max_angle)
    face_chart, C = _compact_ids(ops.uv_chart_ids(adj, label))
    for splits in range(max_splits + 1):
        atlas = Atlas(V, F, face_chart, C, label)
        offs, scale = pack_charts(atlas.box.cpu().numpy(), R, pad)
        vt = ops.uv_place(atlas.uvl, atlas.uv_chart, torch.from_numpy(offs).to(V.device), scale)
        count, bad = ops.uv_coverage(vt, atlas.ft, R)
        if not bool(bad.any()):
            break
        face_chart, C = split_charts(atlas, bad)
    else:
        raise RuntimeError("unwrap: texels still covered twice after %d chart splits" % max_splits)
    uv = atlas.uvl[atlas.ft]          # chart-local fp64: UV area / scale^2 before the fp32 rounding of vt
    e1, e2 = uv[:, 1] - uv[:, 0], uv[:, 2] - uv[:, 0]
    uv_area = 0.5 * (e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0])
    live = area > 0
    stretch = uv_area[live] / area[live]
    smin, smax, cov = torch.stack([stretch.min(), stretch.max(), (count > 0).sum().double()]).tolist()
    info = dict(charts=C, scale=scale, utilisation=cov / float(R * R), stretch_min=smin, stretch_max=smax,
                splits=splits, count=count)
    return vt, atlas.ft, info


def make_uvmap(mesh_path, out_path, faces=30000, resolution=1680, padding=4, max_angle=60., device="cuda"):
    """read_mesh -> simplify -> unwrap -> write_obj.  Returns (simplify info, unwrap info without the coverage)."""
    V, F = read_mesh(mesh_path)
    dev = torch.device(device)
    V, F, sinfo = simplify(V.to(dev), F.to(dev), faces=faces)
    vt, ft, uinfo = unwrap(V, F, resolution=resolution, padding=padding, max_angle=max_angle)
    uinfo.pop("count")
    write_obj(out_path, V, F, vt, ft)
    return sinfo, uinfo


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m selfreconcode_b200.uvmap",
                                 description="<rec-root>/tmp.ply -> <rec-root>/template/uvmap.obj (simplified, UV "
                                             "unwrapped) for texture.bake_from_network")
    ap.add_argument("--rec-root", required=True)
    ap.add_argument("--faces", type=int, default=30000)
    ap.add_argument("--resolution", type=int, default=1680)
    ap.add_argument("--padding", type=int, default=4)
    ap.add_argument("--max-angle", type=float, default=60.)
    ap.add_argument("--gid", type=int, default=0)
    a = ap.parse_args(argv)
    src = osp.join(a.rec_root, "tmp.ply")
    if not osp.isfile(src):
        sys.exit("uvmap: %s is missing: run infer.py on this result directory first" % src)
    out = osp.join(a.rec_root, "template", "uvmap.obj")
    sinfo, uinfo = make_uvmap(src, out, a.faces, a.resolution, a.padding, a.max_angle, "cuda:%d" % a.gid)
    print("uvmap: %s -> %s: %d -> %d faces in %d rounds (%s), %d charts, utilisation %.3f, stretch [%.3f, %.3f]"
          % (src, out, sinfo["faces_in"], sinfo["faces_out"], sinfo["rounds"], sinfo["stop"], uinfo["charts"],
             uinfo["utilisation"], uinfo["stretch_min"], uinfo["stretch_max"]))


if __name__ == "__main__":
    main()
