"""GPU: template simplification and UV atlas (csrc/mesh_simplify.cu, csrc/uv_atlas.cu, uvmap.py) against the float64
twin tests/uvmap_ref.py stage by stage, the invariants of simplify / unwrap on marching-cubes meshes, and
make_uvmap -> bake_from_network end to end."""
import math
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import helpers as H
import uvmap_ref as U

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _mc(fn, n=40, lo=-0.8, hi=0.8):
    from selfreconcode_b200 import ops
    t = torch.linspace(lo, hi, n, dtype=torch.float64)
    x, y, z = torch.meshgrid(t, t, t, indexing="ij")
    g = fn(x, y, z).float().contiguous().to(DEV)
    st = (hi - lo) / (n - 1)
    return ops.marching_cubes(g, st, st, st, lo, lo, lo, 0.0)


def sphere(n=40):
    return _mc(lambda x, y, z: torch.sqrt(x * x + y * y + z * z) - 0.5, n)


def torus(n=48):
    return _mc(lambda x, y, z: torch.sqrt((torch.sqrt(x * x + y * y) - 0.45) ** 2 + z * z) - 0.18, n)


def clipped(n=40):
    # the sphere leaves the grid on +x: an open boundary, and corners marching cubes leaves at -1
    return _mc(lambda x, y, z: torch.sqrt((x - 0.5) ** 2 + y * y + z * z) - 0.55, n)


def two_spheres(n=24):
    V, F = sphere(n)
    i = int(torch.argmax(V[:, 0]))
    V2 = V.clone()
    V2[:, 0] = 2 * V[i, 0] - V[:, 0]          # the mirror image touches the sphere at vertex i
    F2 = F[:, [0, 2, 1]] + V.shape[0]
    F2 = torch.where(F2 == i + V.shape[0], torch.full_like(F2, i), F2)
    return torch.cat([V, V2]), torch.cat([F, F2])


def body():
    import test_gpu_mesh_shade as S
    net, _, _, TmpVs, Tmpfs, _ = S._scene()
    return TmpVs.float().contiguous(), Tmpfs.long().contiguous()


MESHES = {"sphere": sphere, "torus": torus, "clipped": clipped, "two_spheres": two_spheres, "body": body}


def _np(t):
    return t.detach().cpu().numpy()


def _topology_stats(V, F):
    """(Euler characteristic, boundary loops, edges with more than two faces, smallest face area)."""
    F = _np(F)
    E = U.edges(F)
    cnt = {}
    for a, b, c in F:
        for x, y in ((a, b), (b, c), (c, a)):
            k = (min(x, y), max(x, y))
            cnt[k] = cnt.get(k, 0) + 1
    bnd = [k for k, m in cnt.items() if m == 1]
    parent = {}

    def find(x):
        while parent.setdefault(x, x) != x:
            x = parent[x]
        return x
    for a, b in bnd:
        parent[find(a)] = find(b)
    loops = len({find(a) for a, _ in bnd})
    used = np.unique(F)
    Vn = _np(V).astype(np.float64)
    area = np.linalg.norm(np.cross(Vn[F[:, 1]] - Vn[F[:, 0]], Vn[F[:, 2]] - Vn[F[:, 0]]), axis=1)
    return len(used) - len(E) + len(F), loops, sum(m > 2 for m in cnt.values()), area.min()


# ---- 1. one round, stage by stage against the twin ----------------------------------------------------------------
def test_round_vs_twin():
    from selfreconcode_b200 import ops, uvmap
    V, F = sphere(24)
    V, F, _, _ = uvmap.drop_broken(V, F)
    nv = V.shape[0]
    topo = ops.mesh_reg_topology(F, nv)
    csr = uvmap._vertex_face_csr(F, nv)
    Q, fixed = ops.simplify_quadrics(V, F, csr, topo)
    vstar, cost, key = ops.simplify_edge_cost(V, F, csr, topo, Q, fixed)
    sel = ops.simplify_select(topo, key)
    Vn, Fn, E = _np(V), _np(F), _np(topo.edges)
    assert np.array_equal(E, U.edges(Fn))
    Qr = U.quadrics(Vn, Fn)
    iu = np.triu_indices(4)
    Qr10 = Qr[:, iu[0], iu[1]]
    scale = np.abs(Qr10).max(1, keepdims=True)
    assert (np.abs(_np(Q) - Qr10) <= 1e-10 * scale).all()
    fx = U.fixed_vertices(Fn, nv)
    assert np.array_equal(_np(fixed).astype(bool), fx)
    keys = [int(k) & U.NO_KEY for k in _np(key)]
    vs, cs = _np(vstar), _np(cost)
    nvalid = 0
    for e, (a, b) in enumerate(E):
        Qe = Qr[a] + Qr[b]
        v, c, solved = U.solve(Qe, Vn[a].astype(np.float64), Vn[b].astype(np.float64))
        assert abs(cs[e] - c) <= 1e-9 * max(abs(c), np.abs(Qe).max() * np.linalg.norm(Vn[a] - Vn[b]) ** 2), e
        if solved:
            assert np.linalg.norm(vs[e] - v) <= 1e-6 * np.linalg.norm(Vn[a] - Vn[b]), e
        ok, margin = U.edge_checks(Vn, Fn, a, b, vs[e], fx)
        dev_ok = keys[e] != U.NO_KEY
        assert dev_ok == ok or margin < 1e-12, e
        nvalid += dev_ok
        if dev_ok:
            assert keys[e] == U.edge_key(cs[e], e, True)
    assert nvalid > len(E) // 4
    selr = U.select(E, nv, Fn, keys)
    assert np.array_equal(_np(sel).astype(bool), selr) and selr.sum() > 0
    n = int(selr.sum())
    V2, F2 = ops.simplify_collapse(V, F, topo.edges, sel, vstar, nv - n, Fn.shape[0] - 2 * n)
    V2r, F2r = U.collapse(Vn, Fn, E, selr, vs)
    assert np.array_equal(_np(V2), V2r) and np.array_equal(_np(F2), F2r)


def test_atlas_stages_vs_twin():
    from selfreconcode_b200 import ops, uvmap
    V, F = sphere(24)
    V, F, _, _ = uvmap.drop_broken(V, F)
    V, F, _ = uvmap.simplify(V, F, faces=800)
    nv, Fn, Vn = V.shape[0], _np(F), _np(V).astype(np.float64)
    csr = uvmap._vertex_face_csr(F, nv)
    adj = ops.uv_face_adjacency(F, csr)
    assert np.array_equal(_np(adj), U.face_adjacency(Fn, nv))
    normal, area, lab0 = ops.uv_labels(V, F, adj, 60., passes=0)
    lab0r, gap = U.initial_labels(_np(normal), _np(adj))
    tie = gap < 1e-12
    assert np.array_equal(_np(lab0)[~tie], lab0r[~tie])
    _, _, lab = ops.uv_labels(V, F, adj, 60.)
    labr = U.smooth_labels(_np(normal), _np(area), _np(adj), _np(lab0), 60.)
    assert np.array_equal(_np(lab), labr)
    cid = ops.uv_chart_ids(adj, lab)
    assert np.array_equal(_np(cid), U.charts(_np(adj), labr))
    vt, ft, info = uvmap.unwrap(V, F, resolution=128, padding=2)
    fc, C = uvmap._compact_ids(cid)
    at = uvmap.Atlas(V, F, fc, C, lab)
    uvl, uc, uvv, box = _np(at.uvl), _np(at.uv_chart), _np(at.uv_vert), _np(at.box)
    compared = 0
    for c in range(C):
        m = uc == c
        ref, (w, h), tie = U.project_chart(Vn[uvv[m]], int(_np(at.chart_label)[c]), want_tie=True)
        if tie:         # a square box or an isotropic chart: either orientation is the rule's answer
            continue
        assert abs(box[c, 0] - w) <= 1e-9 * w and abs(box[c, 1] - h) <= 1e-9 * w
        assert np.abs(uvl[m] - ref).max() <= 1e-9 * max(w, 1e-30), c
        compared += 1
    assert compared >= C // 2
    # coverage of the final atlas: exact away from edges
    count = _np(info["count"])
    cr, near = U.coverage(_np(vt), _np(ft), 128)
    diff = count != cr
    assert not (diff & (near > 1e-6)).any()
    assert cr.max() <= 1


# ---- 2. simplify invariants ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(MESHES))
def test_simplify_invariants(name):
    from selfreconcode_b200 import ops, uvmap
    V0, F0 = MESHES[name]()
    V0, F0, df, dv = uvmap.drop_broken(V0, F0)
    target = 2000 if name != "body" else 6000
    V, F, info = uvmap.simplify(V0, F0, faces=target)
    print("simplify %s: %s" % (name, {k: v for k, v in info.items() if k != "faces_per_round"}))
    assert F.shape[0] == target or info["stop"] != "target"
    assert F.shape[0] >= target
    chi0, loops0, nm0, _ = _topology_stats(V0, F0)
    chi, loops, nm, amin = _topology_stats(V, F)
    assert (chi, loops) == (chi0, loops0)
    assert nm == nm0 == 0 or nm <= nm0
    assert amin > 0
    topo = ops.mesh_reg_topology(F0, V0.shape[0])
    _, fixed = ops.simplify_quadrics(V0, F0, uvmap._vertex_face_csr(F0, V0.shape[0]), topo)
    P = {tuple(r) for r in _np(V).view(np.int32)}
    for r in _np(V0)[_np(fixed).astype(bool)].view(np.int32):
        assert tuple(r) in P
    V2, F2, _ = uvmap.simplify(V0, F0, faces=target)
    assert torch.equal(V, V2) and torch.equal(F, F2)
    if name == "sphere":
        r = torch.linalg.norm(V.double(), dim=1)
        c = torch.linalg.norm(V.double()[F].mean(1), dim=1)
        assert (r - 0.5).abs().max() < 0.005 and (c - 0.5).abs().max() < 0.01
    if name == "clipped":
        assert df > 0 or loops0 > 0


# ---- 3. unwrap invariants ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sphere", "body"])
def test_unwrap_invariants(name):
    from selfreconcode_b200 import uvmap
    R, pad = 512, 4
    V0, F0 = MESHES[name]()
    V, F, _ = uvmap.simplify(V0, F0, faces=3000)
    vt, ft, info = uvmap.unwrap(V, F, resolution=R, padding=pad, max_angle=60.)
    print("unwrap %s: %s" % (name, {k: v for k, v in info.items() if k != "count"}))
    vtn, ftn = _np(vt).astype(np.float64), _np(ft)
    assert (vtn >= 0).all() and (vtn <= 1).all()
    uv = vtn[ftn]
    e1, e2 = uv[:, 1] - uv[:, 0], uv[:, 2] - uv[:, 0]
    uva = 0.5 * (e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0])
    Vn, Fn = _np(V).astype(np.float64), _np(F)
    n3 = np.cross(Vn[Fn[:, 1]] - Vn[Fn[:, 0]], Vn[Fn[:, 2]] - Vn[Fn[:, 0]])
    a3 = 0.5 * np.linalg.norm(n3, axis=1)
    live = a3 > 1e-12
    assert (uva[live] > 0).all()
    # UV area / 3-D area = s^2 |n . d| per face, d = its chart's direction
    from selfreconcode_b200 import ops
    csr = uvmap._vertex_face_csr(F, V.shape[0])
    adj = ops.uv_face_adjacency(F, csr)
    _, _, lab = ops.uv_labels(V, F, adj, 60.)
    d = U.directions()[_np(lab)]
    s = info["scale"]
    expect = s * s * np.abs((n3 / np.maximum(2 * a3, 1e-300)[:, None] * d).sum(1))
    rel = np.abs(uva / np.maximum(a3, 1e-300) - expect) / expect
    assert rel[live & (a3 > 1e-3 * a3.max())].max() < 1e-4
    assert math.cos(math.radians(60.)) - 1e-6 <= info["stretch_min"] <= info["stretch_max"] <= 1 + 1e-6
    # no texel covered twice under the twin's exact rasterisation
    cr, _ = U.coverage(vtn, ftn, R)
    assert cr.max() <= 1
    # charts at least `padding` texels apart: group UV vertices into charts by ft connectivity of faces
    chart_of_uv = np.full(vtn.shape[0], -1)
    fc, C = uvmap._compact_ids(ops.uv_chart_ids(adj, lab))
    for f, c in zip(ftn, _np(fc)):
        chart_of_uv[f] = c
    lo = np.full((info["charts"], 2), np.inf)
    hi = -lo
    np.minimum.at(lo, chart_of_uv, vtn)
    np.maximum.at(hi, chart_of_uv, vtn)
    for i in range(lo.shape[0]):
        gap = np.maximum(lo - hi[i], lo[i] - hi).max(1)
        gap[i] = np.inf
        assert gap.min() >= pad / R - 1e-6
    assert info["utilisation"] > (0.2 if name == "body" else 0.0)


# ---- 4. end to end ---------------------------------------------------------------------------------------------------
def test_make_uvmap_then_bake(tmp_path, monkeypatch):
    import test_gpu_texture as T
    from selfreconcode_b200 import ops, uvmap
    from selfreconcode_b200.texture import bake_from_network, load_obj_uv
    H.dropin()
    from dataset import write_sequence
    from dataset.dataset import SceneDataset
    from model.raster import screen_vertices
    from model.snapshot import write_ply
    n_frames, side, R = 6, 160, 256
    net, data, cams, TmpVs, Tmpfs = T.scene(side, n_frames)
    res = tmp_path / "result"
    res.mkdir()
    write_ply(str(res / "tmp.ply"), TmpVs, Tmpfs)
    obj = str(res / "template" / "uvmap.obj")
    sinfo, uinfo = uvmap.make_uvmap(str(res / "tmp.ply"), obj, faces=3000, resolution=R, padding=2)
    print("make_uvmap:", sinfo["faces_in"], sinfo["faces_out"], sinfo["stop"], uinfo)
    Vr, Fr, vt, ft = load_obj_uv(obj)
    D = T.deformed(net, data, Vr.to(DEV), list(range(n_frames)))
    imgs, masks = [], []
    for n in range(n_frames):
        p2f, _, _ = ops.raster_mesh(screen_vertices(D[n:n + 1], cams), Fr.to(DEV), side, side)
        hit = p2f[0, ..., 0].cpu().numpy() >= 0
        imgs.append(np.where(hit[..., None], T.smooth_image(n, side), 0).astype(np.float32) / 255. * 2 - 1)
        masks.append(hit.astype(np.float32))
    root = str(tmp_path / "seq")
    f, pp = data.focals.detach().view(2).cpu().numpy(), data.pps.detach().view(2).cpu().numpy()
    write_sequence(root, np.stack(imgs), np.stack(masks), data.poses.detach().cpu().numpy(),
                   data.trans.detach().cpu().numpy(), np.zeros(10, np.float32),
                   dict(fx=f[0], fy=f[1], cx=pp[0], cy=pp[1], quat=[0., 0., 0., 1.], T=[0., 0., 0.]))
    ds = SceneDataset(root, {'deformer': 128})
    with torch.no_grad():
        ds.conds[0].copy_(data.conds[0].detach().cpu())
    onet = types.SimpleNamespace(deformer=net.deformer, dataset=ds)
    out = bake_from_network(onet, obj, str(tmp_path / "tex"), num=n_frames, resolution=R, min_views=2)
    count, _ = ops.uv_coverage(vt.to(DEV), ft.to(DEV), R, want_bad=False)
    _, near = U.coverage(_np(vt), _np(ft), R)
    diff = _np(out["tex_mask"]) != (_np(count) > 0)
    # the bake's UV raster works in fp32 at coordinates up to R, so it may decide differently within ~1e-3 texel
    # of an edge; the coverage kernel's decisions are exact
    assert not (diff & (near > 1e-3)).any(), int(diff.sum())
    assert bool(out["mask_final"].any())
    # the CLI on the same directory
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    r = subprocess.run([sys.executable, "-m", "selfreconcode_b200.uvmap", "--rec-root", str(res), "--faces", "3000",
                        "--resolution", str(R), "--padding", "2"], env=env, capture_output=True, text=True, cwd=H.ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "uvmap:" in r.stdout
    assert load_obj_uv(obj)[2].shape == vt.shape
    r = subprocess.run([sys.executable, "-m", "selfreconcode_b200.uvmap", "--rec-root", str(tmp_path / "none")],
                       env=env, capture_output=True, text=True, cwd=H.ROOT)
    assert r.returncode != 0 and "infer.py" in r.stderr


def test_invalid_arguments():
    from selfreconcode_b200 import uvmap
    V, F = sphere(16)
    with pytest.raises(ValueError):
        uvmap.unwrap(V, F, max_angle=30.)
    with pytest.raises(ValueError):
        uvmap.unwrap(V, F, max_angle=85.)
    with pytest.raises(RuntimeError):
        uvmap.simplify(V.cpu(), F.cpu())
