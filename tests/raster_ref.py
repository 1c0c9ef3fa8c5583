"""Float64 restatement of the mesh rasteriser (csrc/raster.cu, ops.raster_mesh; oracle.raster_mesh is its fp32 twin).

The rule
--------
Screen vertices are (col, row, view depth z) per frame, pixel centres at integers: pixel (r, c) is the point (c, r).
A face (v0, v1, v2) is dropped when a vertex is not finite, when any z <= 1e-8, or when its area
    A = e(v1, v2; v0),     e(a, b; p) = (xa - px)(yb - py) - (xb - px)(ya - py),
has |A| < 1e-12 (both thresholds are the fp32 constants the kernel compares with).  At a pixel centre p its edge values
are w0 = e(v1, v2; p), w1 = e(v2, v0; p), w2 = e(v0, v1; p) and l_i = w_i / A.  Coverage is inclusive: the face covers p
when all l_i >= 0 (winding does not matter).  Barycentrics are perspective-correct: q_i = l_i / z_i, b = q / sum(q), and
the depth is z = 1 / sum(q).  The covering face of least depth wins; an exact depth tie goes to the lowest face id.  With
N frames sharing the faces, frame n's face f has id n F + f.  Empty pixels hold id -1, barycentrics -1 and depth -1.
The restatement computes this in float64 from the fp32 vertex values the kernel reads.  Coordinates are assumed small
enough that no product overflows fp32 (|x|, |y| up to ~1e9 at the screen sizes used).

How far the kernel may stray from it
------------------------------------
The kernel evaluates the same formula in fp32 with every operation rounded once (no contraction), u = 2^-24.  For
e(a, b; p): each of the four differences, each of the two products and the final difference rounds once, so
    |fl(e) - e| <= gamma_4 (|(xa - px)(yb - py)| + |(xb - px)(ya - py)|),     gamma_4 = 4u / (1 - 4u),
and the bound is 0 when every intermediate is an fp32 number (then the kernel's value is exact).  The same holds for A.
Propagated to first order through l_i = fl(w_i fl(1/A)), q_i = fl(l_i / z_i), s = fl(fl(q0 + q1) + q2),
b_i = fl(q_i / s) and z = fl(1 / s):
    e_l = (e_w + |l| e_A) / |A| + 2u |l|        e_q = e_l / z_i + u |q|        e_s = sum e_q + 2u sum |q|
    e_b = e_q / s + |q| e_s / s^2 + u |b|       e_z = e_s / s^2 + u z
times 1.01 for the neglected higher-order terms (they are below 1e-3 of the first-order ones because a face whose
e_A exceeds |A| / 1000 is treated as uncertain).  Nothing here is fitted to the kernel's output.

Per pixel classification
------------------------
An edge value is *certain* when |w| > e_w or e_w = 0 (the kernel's sign then equals the exact one), *near* when
|w| <= e_w.  A fragment (face, pixel in its bounding box) is certainly covered when its area is certainly kept and all
three edge values are certain and covering; it is excluded when it certainly is not; otherwise it *may* be covered.
- sensitive: a may-be fragment whose depth range reaches the nearest certain fragment's, or another certain fragment
  whose depth range reaches the nearest one's (not counting bit-identical duplicate faces, whose fp32 depths
  tie exactly and go to the lower id on both sides).  Everywhere else the kernel must make the float64 choice.
- must_cover: the pixel is near an edge (same fp32 endpoints) of two faces on opposite sides of it, each with its other
  two edge values certain and covering.  The kernel's edge values of the two faces are then exact negations (or equal,
  for opposite windings), so one of the two covers the pixel: it may never be -1 there.
- outline: near an edge of a fragment that is not excluded, and not must_cover (silhouettes, vertices).
"""
import numpy as np

U = 2.0 ** -24
GAMMA4 = 4 * U / (1 - 4 * U)
Z_MIN = float(np.float32(1e-8))
A_MIN = float(np.float32(1e-12))
SAFETY = 1.01
EDGES = ((1, 2), (2, 0), (0, 1))       # w_k = e(v_a, v_b; p)


def _is_f32(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return x.astype(np.float32).astype(np.float64) == x


def _diff(a, b):
    """a - b in float64 and whether it is the exact difference and an fp32 number (the kernel's is then exact)."""
    d = a - b
    return d, _is_f32(d) & (d + b == a) & (a - d == b)


def edge(xa, ya, xb, yb, px, py):
    """-> (e(a, b; p) in float64, bound on |fp32 kernel value - e|)."""
    d1, x1 = _diff(xa, px)
    d2, x2 = _diff(yb, py)
    d3, x3 = _diff(xb, px)
    d4, x4 = _diff(ya, py)
    p1, p2 = d1 * d2, d3 * d4
    w = p1 - p2
    mag = np.abs(p1) + np.abs(p2)
    exact = x1 & x2 & x3 & x4 & _is_f32(p1) & _is_f32(p2) & _is_f32(w)
    # 2^-50 mag covers float64's own rounding of p1, p2 and w
    return w, np.where(exact, 0., GAMMA4 * mag + 2.0 ** -50 * mag)


class Result:
    """face [N,H,W] int64 (n F + f or -1), bary [N,H,W,3] and zbuf [N,H,W] (-1 where empty), float64; bary_bound
    [N,H,W,3] and z_bound [N,H,W] (the fp32 bound of the chosen face, 0 where empty); sensitive, must_cover, outline
    [N,H,W] bool."""


def raster(verts, faces, H, W, chunk=1 << 21):
    vs = np.asarray(verts, np.float32)
    if vs.ndim == 2:
        vs = vs[None]
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    N, V = vs.shape[:2]
    F = fc.shape[0]
    P = H * W
    out = Result()
    out.face = -np.ones((N, H, W), np.int64)
    out.bary = -np.ones((N, H, W, 3))
    out.zbuf = -np.ones((N, H, W))
    out.bary_bound = np.zeros((N, H, W, 3))
    out.z_bound = np.zeros((N, H, W))
    for k in ("sensitive", "must_cover", "outline"):
        setattr(out, k, np.zeros((N, H, W), bool))
    if N == 0 or F == 0:
        return out
    T = vs.astype(np.float64)[:, fc]                      # [N,F,3 vertices,3]
    x, y, z = T[..., 0], T[..., 1], T[..., 2]
    finite = np.isfinite(T).all((2, 3))
    with np.errstate(invalid="ignore", over="ignore"):
        zok = finite & (z > Z_MIN).all(2)
        A, eA = edge(x[..., 1], y[..., 1], x[..., 2], y[..., 2], x[..., 0], y[..., 0])
        aA = np.abs(A)
        keep = zok & (aA >= A_MIN)                        # the rule's decision
        keep_sure = zok & (aA - eA >= A_MIN) & (eA <= 1e-3 * aA)
        maybe_kept = zok & (aA + eA >= A_MIN)
    # edge ids per frame: an edge is its two fp32 endpoints (x, y), in a canonical order; orient = +1 when the face's
    # slot runs along that order
    ea = np.stack([np.stack([x[..., a], y[..., a]], -1) for a, _ in EDGES], 2)      # [N,F,3,2]
    eb = np.stack([np.stack([x[..., b], y[..., b]], -1) for _, b in EDGES], 2)
    fwd = (ea[..., 0] < eb[..., 0]) | ((ea[..., 0] == eb[..., 0]) & (ea[..., 1] <= eb[..., 1]))
    lo = np.where(fwd[..., None], ea, eb)
    hi = np.where(fwd[..., None], eb, ea)
    nn = np.broadcast_to(np.arange(N, dtype=np.float64)[:, None, None, None], fwd.shape + (1,))
    rows = np.concatenate([nn, lo, hi], -1).reshape(-1, 5)
    rows = np.where(np.isfinite(rows), rows, 0.)
    _, eid = np.unique(rows, axis=0, return_inverse=True)
    eid = eid.reshape(N, F, 3)
    orient = np.where(fwd, 1, -1)

    with np.errstate(invalid="ignore"):
        xmin, xmax = np.where(finite, x.min(2), 0.), np.where(finite, x.max(2), -1.)
        ymin, ymax = np.where(finite, y.min(2), 0.), np.where(finite, y.max(2), -1.)
    c0 = np.maximum(0, np.ceil(np.clip(xmin, -1, W))).astype(np.int64)
    c1 = np.minimum(W - 1, np.floor(np.clip(xmax, -1, W))).astype(np.int64)
    r0 = np.maximum(0, np.ceil(np.clip(ymin, -1, H))).astype(np.int64)
    r1 = np.minimum(H - 1, np.floor(np.clip(ymax, -1, H))).astype(np.int64)
    live = maybe_kept & (c1 >= c0) & (r1 >= r0)
    pn, pf = np.nonzero(live)
    cnt = (c1 - c0 + 1)[pn, pf] * (r1 - r0 + 1)[pn, pf]

    # fragment lists, concatenated over chunks
    keys = dict(pix=[], fid=[], z=[], cert=[], exact=[], zlo=[], zhi=[], ez=[], b=[], eb=[], near=[], vtx=[])
    mc_keys = []
    ends = np.cumsum(cnt)
    start = 0
    while start < len(pn):
        stop = max(start + 1, int(np.searchsorted(ends, (ends[start - 1] if start else 0) + chunk, "right")))
        sel = slice(start, stop)
        n, f, m = pn[sel], pf[sel], cnt[sel]
        j = np.repeat(np.arange(len(n)), m)
        off = np.arange(m.sum()) - np.repeat(np.cumsum(m) - m, m)
        n, f = n[j], f[j]
        wd = (c1 - c0 + 1)[n, f]
        r = r0[n, f] + off // wd
        c = c0[n, f] + off % wd
        px, py = c.astype(np.float64), r.astype(np.float64)
        X, Y, Z = x[n, f], y[n, f], z[n, f]
        Af, eAf = A[n, f], eA[n, f]
        w, ew = [], []
        for a, b in EDGES:
            wk, ek = edge(X[:, a], Y[:, a], X[:, b], Y[:, b], px, py)
            w.append(wk)
            ew.append(ek)
        w, ew = np.stack(w, 1), np.stack(ew, 1)
        sA = np.sign(Af)[:, None]
        cert = (np.abs(w) > ew) | (ew == 0)
        near = np.abs(w) <= ew
        pos = sA * w >= 0
        ks, kk = keep_sure[n, f], keep[n, f]
        cov_sure = ks & (cert & pos).all(1)
        cov_exact = kk & pos.all(1)
        excl = np.where(ks, (cert & ~pos).any(1),
                        (cert & (w > 0)).any(1) & (cert & (w < 0)).any(1))
        excl |= ~maybe_kept[n, f]
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            aA_ = np.abs(Af)[:, None]
            l = w / Af[:, None]
            el = (ew + np.abs(l) * eAf[:, None]) / aA_ + 2 * U * np.abs(l)
            q = l / Z
            eq = el / Z + U * np.abs(q)
            s = np.sort(q, 1).sum(1)       # in a fixed order, so that a face's depth does not depend on its winding
            es = eq.sum(1) + 2 * U * np.abs(q).sum(1)
            zf = 1. / s
            bf = q / s[:, None]
            eb_ = SAFETY * (eq / np.abs(s)[:, None] + np.abs(q) * (es / (s * s))[:, None] + U * np.abs(bf))
            ez = SAFETY * (es / (s * s) + U * np.abs(zf))
            ok = np.isfinite(zf) & (s > 0) & np.isfinite(ez) & ks
            zlo = np.where(ok, zf - ez, 0.)
            zhi = np.where(ok, zf + ez, np.inf)
        rel = ~excl
        g = n * P + r * W + c
        keys["pix"].append(g[rel])
        keys["fid"].append(f[rel])
        keys["z"].append(np.where(cov_exact, zf, np.inf)[rel])
        keys["cert"].append(cov_sure[rel])
        keys["exact"].append(cov_exact[rel])
        keys["zlo"].append(zlo[rel])
        keys["zhi"].append(zhi[rel])
        keys["ez"].append(ez[rel])
        keys["b"].append(bf[rel])
        keys["eb"].append(eb_[rel])
        keys["near"].append(near.any(1)[rel])
        keys["vtx"].append(T[n, f].reshape(-1, 9)[rel])
        # must-cover candidates: edge k near, the other two certain and covering, area certainly kept
        cp = cert & pos
        for k in range(3):
            o1, o2 = [i for i in range(3) if i != k]
            cand = ks & near[:, k] & cp[:, o1] & cp[:, o2]
            side = (orient[n, f, k] * sA[:, 0] > 0)[cand]
            mc_keys.append(np.stack([g[cand], eid[n, f, k][cand], side.astype(np.int64)], 1))
        start = stop

    fr = {k: np.concatenate(v) if v else np.zeros(0) for k, v in keys.items()}
    flat = lambda a: a.reshape(N * P, *a.shape[3:])          # noqa: E731
    if len(fr["pix"]):
        pix = fr["pix"]
        # float64 choice: nearest exactly covering fragment, ties to the lowest id
        cov = fr["exact"]
        o = np.lexsort((fr["fid"][cov], fr["z"][cov], pix[cov]))
        pc = pix[cov][o]
        first = np.r_[True, pc[1:] != pc[:-1]] if len(pc) else np.zeros(0, bool)
        win = np.nonzero(cov)[0][o][first]
        gp = pix[win]
        flat(out.face)[gp] = (gp // P) * F + fr["fid"][win]
        flat(out.bary)[gp] = fr["b"][win]
        flat(out.zbuf)[gp] = fr["z"][win]
        flat(out.bary_bound)[gp] = fr["eb"][win]
        flat(out.z_bound)[gp] = fr["ez"][win]
        # nearest and runner-up certain fragments by (depth, id)
        ct = fr["cert"]
        zc = np.where(ct, fr["z"], np.inf)
        o = np.lexsort((fr["fid"], zc, pix))
        ps = pix[o]
        first = np.r_[True, ps[1:] != ps[:-1]]
        grp = np.cumsum(first) - 1
        best = o[first]
        zhi_best = np.full(N * P, np.inf)
        has = ct[best]
        zhi_best[pix[best[has]]] = fr["zhi"][best[has]]
        sens = np.zeros(N * P, bool)
        # may-be fragments that reach the nearest certain one
        mb = ~ct
        sens[pix[mb][fr["zlo"][mb] <= zhi_best[pix[mb]]]] = True
        # runner-up certain fragments within the depth bound
        rank = np.arange(len(o)) - np.flatnonzero(first)[grp]
        run = o[rank >= 1]
        run = run[ct[run]]                 # certain fragments sort first, so their pixel's nearest one is certain too
        bi = np.full(N * P, -1, np.int64)
        bi[pix[best[has]]] = best[has]
        rb = bi[pix[run]]
        gap_close = fr["z"][run] - fr["ez"][run] <= fr["z"][rb] + fr["ez"][rb]
        twin = (fr["z"][run] == fr["z"][rb]) & (fr["vtx"][run] == fr["vtx"][rb]).all(1)
        sens[pix[run][gap_close & ~twin]] = True
        flat(out.sensitive)[:] = sens
        # must-cover: both sides of one edge at one pixel
        mk = np.concatenate(mc_keys) if mc_keys else np.zeros((0, 3), np.int64)
        if len(mk):
            u, inv = np.unique(mk[:, :2], axis=0, return_inverse=True)
            sides = np.zeros((len(u), 2), bool)
            sides[inv.reshape(-1), mk[:, 2]] = True
            both = sides.all(1)
            flat(out.must_cover)[u[both, 0]] = True
        nr = np.zeros(N * P, bool)
        nr[pix[fr["near"]]] = True
        flat(out.outline)[:] = nr & ~flat(out.must_cover)
    return out


# ---- scenes ----------------------------------------------------------------------------------------------------------
_DIRS = np.array([(1, 1), (1, 2), (2, 1), (1, 3), (3, 1), (2, 3), (3, 2)], np.float64)


def crack_scene(grid, n_frames, seed, cell=7):
    """Disjoint quads, one per cell x cell block of a (grid cell)^2 screen, each split into two faces along a diagonal
    that passes through the block's centre pixel (and through further pixel centres when its integer direction is
    short) in real arithmetic.  The diagonal's endpoints lie at random distances along it and are rounded to fp32, so
    the rounded edge passes within rounding of those centres; a fifth of the quads per frame get endpoints that are fp32
    numbers (the centres then lie exactly on the edge).  The two other corners lie on either side.  Every third quad's
    second face has the opposite winding.  Per-vertex depths are random in [1, 3].
    -> (verts [N, 4 Q, 3] float32, faces [2 Q, 3] int64, side); faces 2i and 2i + 1 form quad i."""
    rng = np.random.default_rng(seed)
    Q = grid * grid
    side = grid * cell
    i = np.arange(Q)
    base = (i % grid) * cell, (i // grid) * cell
    P = np.stack([base[0] + cell // 2, base[1] + cell // 2], 1).astype(np.float64)
    reach = (cell - 1) / 2 - 0.1                    # corners stay inside the block
    verts = np.zeros((n_frames, 4 * Q, 3), np.float32)
    for n in range(n_frames):
        d = _DIRS[rng.integers(0, len(_DIRS), Q)] * rng.choice([-1., 1.], (Q, 2))
        dl = np.linalg.norm(d, axis=1, keepdims=True)
        t = rng.uniform(0.35, 1.0, (Q, 2)) * reach / dl
        exact = rng.random(Q) < 0.2
        t[exact] = np.round(t[exact] * 4) / 4
        a = P + t[:, :1] * d
        b = P - t[:, 1:] * d
        nrm = np.stack([-d[:, 1], d[:, 0]], 1) / dl
        h = rng.uniform(0.5, 1.0, (Q, 2)) * reach
        c = P + h[:, :1] * nrm
        e = P - h[:, 1:] * nrm
        xy = np.stack([a, b, c, e], 1).reshape(-1, 2)
        verts[n, :, :2] = xy
        verts[n, :, 2] = rng.uniform(1., 3., 4 * Q)
    f0 = np.stack([4 * i, 4 * i + 1, 4 * i + 2], 1)
    f1 = np.where((i % 3 == 2)[:, None], np.stack([4 * i, 4 * i + 1, 4 * i + 3], 1),
                  np.stack([4 * i + 1, 4 * i, 4 * i + 3], 1))
    faces = np.stack([f0, f1], 1).reshape(-1, 3).astype(np.int64)
    return verts, faces, side


def fp32_raster(verts, faces, H, W, strict=False, screen_bary=False, ties_to_last=False, contract=False):
    """The kernel's fp32 arithmetic (oracle.raster_mesh's, vectorised over fragments) with switches that each break one
    part of the rule, for negative controls: strict (> 0 coverage), screen_bary (no perspective correction),
    ties_to_last (an exact depth tie goes to the highest id), contract (each edge function as an FFMA
    fma(a, b, -fl(c d)), the contraction nvcc makes without __fmul_rn / __fsub_rn).  -> (face [N,H,W] int64 n F + f or
    -1, bary [N,H,W,3] float32, zbuf [N,H,W] float32)."""
    f32 = np.float32
    vs = np.asarray(verts, f32)
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    N, F, P = vs.shape[0], fc.shape[0], H * W
    face = -np.ones(N * P, np.int64)
    bary = -np.ones((N * P, 3), f32)
    zbuf = -np.ones(N * P, f32)
    T = vs[:, fc]
    x, y, z = T[..., 0], T[..., 1], T[..., 2]

    def e(xa, ya, xb, yb, px, py):
        a, b, c, d = xa - px, yb - py, xb - px, ya - py
        if contract:
            return (a.astype(np.float64) * b - (c * d).astype(np.float64)).astype(f32)
        return a * b - c * d

    with np.errstate(all="ignore"):
        ok = np.isfinite(T).all((2, 3)) & (z > f32(1e-8)).all(2)
        A = e(x[..., 1], y[..., 1], x[..., 2], y[..., 2], x[..., 0], y[..., 0])
        ok &= np.abs(A) >= f32(1e-12)
        c0 = np.maximum(0, np.ceil(np.where(ok, x.min(2), 0))).astype(np.int64)
        c1 = np.minimum(W - 1, np.floor(np.where(ok, x.max(2), -1))).astype(np.int64)
        r0 = np.maximum(0, np.ceil(np.where(ok, y.min(2), 0))).astype(np.int64)
        r1 = np.minimum(H - 1, np.floor(np.where(ok, y.max(2), -1))).astype(np.int64)
    ok &= (c1 >= c0) & (r1 >= r0)
    n, f = np.nonzero(ok)
    m = (c1 - c0 + 1)[n, f] * (r1 - r0 + 1)[n, f]
    j = np.repeat(np.arange(len(n)), m)
    off = np.arange(m.sum()) - np.repeat(np.cumsum(m) - m, m)
    n, f = n[j], f[j]
    wd = (c1 - c0 + 1)[n, f]
    r, c = r0[n, f] + off // wd, c0[n, f] + off % wd
    px, py = c.astype(f32), r.astype(f32)
    X, Y, Z = x[n, f], y[n, f], z[n, f]
    with np.errstate(all="ignore"):
        inv = f32(1) / A[n, f]
        l = np.stack([e(X[:, a], Y[:, a], X[:, b], Y[:, b], px, py) * inv for a, b in EDGES], 1)
        inside = (l > 0).all(1) if strict else (l >= 0).all(1)
        q = l if screen_bary else l / Z
        s = q[:, 0] + q[:, 1] + q[:, 2]
        inside &= s > 0
        zz = f32(1) / (s if not screen_bary else (l / Z).sum(1, dtype=f32))
        b = q / s[:, None]
    g = (n * P + r * W + c)[inside]
    fid = f[inside]
    key = zz[inside].view(np.uint32).astype(np.int64)
    o = np.lexsort((-fid if ties_to_last else fid, key, g))
    gs = g[o]
    first = np.r_[True, gs[1:] != gs[:-1]] if len(gs) else np.zeros(0, bool)
    win = np.nonzero(inside)[0][o][first]
    gp = gs[first]
    face[gp] = (gp // P) * F + f[win]
    bary[gp] = b[win]
    zbuf[gp] = zz[win]
    return face.reshape(N, H, W), bary.reshape(N, H, W, 3), zbuf.reshape(N, H, W)
