"""Float64 numpy restatement of the template simplification and UV atlas rules (csrc/mesh_simplify.cu,
csrc/uv_atlas.cu, selfreconcode_b200/uvmap.py), one stage at a time.  Each stage takes the engine's decisions of the
stages before it (its keys, selection, v*, labels or UVs) so that a difference points at one rule."""
import math

import numpy as np

SINGULAR_REL = 1e-6
NO_KEY = (1 << 64) - 1


def vertex_faces(F, nv):
    """Each vertex's faces, ascending."""
    out = [[] for _ in range(nv)]
    for f, row in enumerate(np.asarray(F)):
        for v in sorted(set(int(x) for x in row)):
            out[v].append(f)
    return out


def neighbours(F, nv):
    """Each vertex's neighbours, ascending."""
    out = [set() for _ in range(nv)]
    for a, b, c in np.asarray(F):
        for x, y in ((a, b), (b, c), (c, a)):
            if x != y:
                out[x].add(int(y))
                out[y].add(int(x))
    return [sorted(s) for s in out]


def edges(F):
    """Unique edges (a < b), ascending by (a, b)."""
    s = set()
    for a, b, c in np.asarray(F):
        for x, y in ((a, b), (b, c), (c, a)):
            s.add((int(min(x, y)), int(max(x, y))))
    return np.array(sorted(s), dtype=np.int64).reshape(-1, 2)


def face_quadric(p0, p1, p2):
    """Area-weighted plane quadric [4,4] of a triangle (0 at zero area)."""
    n = np.cross(p1 - p0, p2 - p0)
    ln = np.linalg.norm(n)
    if ln == 0:
        return np.zeros((4, 4))
    u = n / ln
    p = np.append(u, -u @ p0)
    return 0.5 * ln * np.outer(p, p)


def quadrics(V, F):
    """Q [V,4,4]: the sum over each vertex's faces, in ascending face order."""
    V = np.asarray(V, np.float64)
    F = np.asarray(F)
    Q = np.zeros((V.shape[0], 4, 4))
    for v, fs in enumerate(vertex_faces(F, V.shape[0])):
        for f in fs:
            Q[v] += face_quadric(*V[F[f]])
    return Q


def fixed_vertices(F, nv):
    """A vertex is fixed unless all its edges have two faces, none of its faces repeats an index, and its faces form
    one closed fan."""
    F = np.asarray(F)
    vf, nb = vertex_faces(F, nv), neighbours(F, nv)
    fixed = np.zeros(nv, bool)
    for v in range(nv):
        fs = vf[v]
        if not fs or any(len(set(F[f])) < 3 for f in fs):
            fixed[v] = True
            continue
        if any(sum(u in F[f] for f in fs) != 2 for u in nb[v]):
            fixed[v] = True
            continue
        row = list(F[fs[0]])
        x, cur, n = row[(row.index(v) + 1) % 3], fs[0], 0
        while True:
            nxt = [f for f in fs if f != cur and x in F[f]][0]
            x = [y for y in F[nxt] if y != v and y != x][0]
            cur, n = nxt, n + 1
            if cur == fs[0] or n > len(fs):
                break
        fixed[v] = n != len(fs)
    return fixed


def qeval(Q, p):
    h = np.append(p, 1.0)
    return h @ Q @ h


def solve(Q, pa, pb):
    """(v*, cost, solved): -A^-1 b when det A > 1e-6 (tr A / 3)^3, else the best of a, b, midpoint (first on ties)."""
    A, b = Q[:3, :3], Q[:3, 3]
    t3 = np.trace(A) / 3.0
    det = np.linalg.det(A)
    if t3 > 0 and det > SINGULAR_REL * t3 ** 3:
        v = -np.linalg.solve(A, b)
        return v, max(qeval(Q, v), 0.0), True
    best = None
    for p in (pa, pb, 0.5 * (pa + pb)):
        c = qeval(Q, p)
        if best is None or c < best[1]:
            best = (p, c)
    return best[0], max(best[1], 0.0), False


def edge_checks(V, F, a, b, vstar, fixed):
    """(valid, smallest |flip dot| relative to |n0| |n1|) of collapsing (a, b) to fp32(vstar)."""
    V = np.asarray(V, np.float64)
    F = np.asarray(F)
    nb = neighbours(F, V.shape[0])
    if fixed[a] or fixed[b]:
        return False, np.inf
    common = sorted(set(nb[a]) & set(nb[b]))
    if len(common) != 2 or any(len(nb[o]) < 4 for o in common):
        return False, np.inf
    vf32 = np.asarray(vstar, np.float32).astype(np.float64)
    ok, margin = True, np.inf
    vf = vertex_faces(F, V.shape[0])
    for w in (a, b):
        for f in vf[w]:
            if a in F[f] and b in F[f]:
                continue
            p = V[F[f]]
            r = p.copy()
            r[list(F[f]).index(w)] = vf32
            n0 = np.cross(p[1] - p[0], p[2] - p[0])
            n1 = np.cross(r[1] - r[0], r[2] - r[0])
            d, s0, s1 = n0 @ n1, n0 @ n0, n1 @ n1
            if s0 > 0 and s1 > 0:
                margin = min(margin, abs(d) / math.sqrt(s0 * s1))
            if not (s1 > 0 and (s0 == 0 or d > 0)):
                ok = False
    return ok, margin


def edge_key(cost, e, valid):
    if not valid:
        return NO_KEY
    return (int(np.array(cost, np.float32).view(np.uint32)) << 32) | int(e)


def select(E, nv, F, keys):
    """Given keys [E] (python ints), the selected edges: key = min over both endpoints' two rings."""
    nb = neighbours(F, nv)
    m1 = [NO_KEY] * nv
    for e, (a, b) in enumerate(E):
        m1[a] = min(m1[a], keys[e])
        m1[b] = min(m1[b], keys[e])
    m2 = [min([m1[v]] + [m1[u] for u in nb[v]]) for v in range(nv)]
    return np.array([keys[e] != NO_KEY and keys[e] == m2[a] == m2[b] for e, (a, b) in enumerate(E)], bool)


def collapse(V, F, E, sel, vstar):
    """Given the selection and v*: b -> a, a at fp32(v*), faces with a repeated corner removed, survivors compacted in
    ascending order."""
    V = np.asarray(V, np.float32).copy()
    F = np.asarray(F)
    remap = np.arange(V.shape[0])
    for e in np.nonzero(sel)[0]:
        a, b = E[e]
        remap[b] = a
        V[a] = np.asarray(vstar[e], np.float32)
    R = remap[F]
    alive = (R[:, 0] != R[:, 1]) & (R[:, 1] != R[:, 2]) & (R[:, 0] != R[:, 2])
    keep = remap == np.arange(V.shape[0])
    new = np.cumsum(keep) - 1
    return V[keep], new[R[alive]]


# ---------------------------------------------------------------------------------------------------------------- atlas
def directions():
    d = [(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1) if (i, j, k) != (0, 0, 0)]
    d = np.array(d, np.float64)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def face_adjacency(F, nv):
    """adj [F,3]: the face across the edge opposite corner k when that edge has exactly two faces, else -1."""
    F = np.asarray(F)
    vf = vertex_faces(F, nv)
    adj = -np.ones((F.shape[0], 3), np.int64)
    for f in range(F.shape[0]):
        for k in range(3):
            a, b = F[f, (k + 1) % 3], F[f, (k + 2) % 3]
            o = [g for g in vf[a] if g != f and b in F[g]]
            if len(o) == 1:
                adj[f, k] = o[0]
    return adj


def initial_labels(normals, adj):
    """argmax_L n . d_L (lowest L on ties); a zero normal takes its lowest-id neighbour's with a normal (else 0).
    -> (labels, gap between the top two dots per face)."""
    D = directions()
    dots = normals @ D.T
    lab = np.argmax(dots, 1)
    srt = np.sort(dots, 1)
    gap = srt[:, -1] - srt[:, -2]
    zero = ~np.any(normals != 0, 1)
    base = lab.copy()
    for f in np.nonzero(zero)[0]:
        nbs = sorted(g for g in adj[f] if g >= 0 and not zero[g])
        base[f] = lab[nbs[0]] if nbs else 0
        gap[f] = gap[nbs[0]] if nbs else np.inf
    return base, gap


def smooth_labels(normals, area, adj, labels, max_angle, passes=8):
    D = directions()
    cmax = math.cos(math.radians(float(np.float32(max_angle))))
    lab = labels.copy()
    for _ in range(passes):
        new = lab.copy()
        for f in range(lab.shape[0]):
            ids = [f] + [int(g) for g in adj[f]]
            labs = [lab[i] if i >= 0 else -1 for i in ids]
            best, bs = lab[f], -1.0
            for L in labs:
                if L < 0 or normals[f] @ D[L] < cmax:
                    continue
                s = 0.0
                for i, l2 in zip(ids, labs):
                    if l2 == L:
                        s += area[i]
                if s > bs or (s == bs and L < best):
                    best, bs = L, s
            new[f] = best
        lab = new
    return lab


def charts(adj, labels):
    """Chart id per face = the minimum face id of its component (same label across two-face edges)."""
    n = labels.shape[0]
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for f in range(n):
        for g in adj[f]:
            if g >= 0 and labels[g] == labels[f]:
                a, b = find(f), find(int(g))
                if a != b:
                    parent[max(a, b)] = min(a, b)
    return np.array([find(f) for f in range(n)], np.int64)


def project_chart(P, label, want_tie=False):
    """Chart-local coordinates [n,2] of the points P [n,3] and the box (w, h); with want_tie also whether the
    principal angle or the landscape turn is a near-tie (within 1e-9), where rounding may pick the other side."""
    d = directions()[label]
    k = int(np.argmin(np.abs(d)))
    t1 = np.cross(d, np.eye(3)[k])
    t1 /= np.linalg.norm(t1)
    t2 = np.cross(d, t1)
    xy = np.stack([P @ t1, P @ t2], 1)
    xy = xy - xy.mean(0)
    cxx, cxy, cyy = (xy[:, 0] ** 2).sum(), (xy[:, 0] * xy[:, 1]).sum(), (xy[:, 1] ** 2).sum()
    th = 0.5 * math.atan2(2 * cxy, cxx - cyy)
    c, s = math.cos(th), math.sin(th)
    uv = np.stack([c * xy[:, 0] + s * xy[:, 1], -s * xy[:, 0] + c * xy[:, 1]], 1)
    w, h = np.ptp(uv[:, 0]), np.ptp(uv[:, 1])
    tie = abs(w - h) <= 1e-9 * max(w, h) or math.hypot(2 * cxy, cxx - cyy) <= 1e-9 * (cxx + cyy)
    if h > w:
        uv = np.stack([-uv[:, 1], uv[:, 0]], 1)
        w, h = h, w
    if want_tie:
        return uv - uv.min(0), (w, h), tie
    return uv - uv.min(0), (w, h)


def _edge_fn(p, q, t):
    if q[0] < p[0] or (q[0] == p[0] and q[1] < p[1]):
        return -_edge_fn(q, p, t)
    return (q[0] - p[0]) * (t[1] - p[1]) - (q[1] - p[1]) * (t[0] - p[0])


def coverage(vt, ft, R):
    """count [R,R] of UV faces covering each texel centre (half-open rule of csrc/uv_atlas.cu) and the distance in
    texels from each centre to its nearest covering-candidate edge (inf where no face is near)."""
    vt = np.asarray(vt, np.float32).astype(np.float64)
    X, Y = vt[:, 0] * R - 0.5, (1.0 - vt[:, 1]) * R - 0.5
    count = np.zeros((R, R), np.int64)
    near = np.full((R, R), np.inf)
    for f in np.asarray(ft):
        P = [(X[i], Y[i]) for i in f]
        a = _edge_fn(P[0], P[1], P[2])
        xs, ys = [p[0] for p in P], [p[1] for p in P]
        c0, c1 = max(0, math.ceil(min(xs)) - 1), min(R - 1, math.floor(max(xs)) + 1)
        r0, r1 = max(0, math.ceil(min(ys)) - 1), min(R - 1, math.floor(max(ys)) + 1)
        for r in range(r0, r1 + 1):
            for c in range(c0, c1 + 1):
                t = (float(c), float(r))
                for k in range(3):
                    p, q = P[k], P[(k + 1) % 3]
                    ln = math.hypot(q[0] - p[0], q[1] - p[1])
                    if ln > 0:
                        near[r, c] = min(near[r, c], _seg_dist(p, q, t))
                if a == 0:
                    continue
                sg = 1.0 if a > 0 else -1.0
                inside = True
                for k in range(3):
                    p, q = P[k], P[(k + 1) % 3]
                    w = sg * _edge_fn(p, q, t)
                    dx, dy = sg * (q[0] - p[0]), sg * (q[1] - p[1])
                    if w < 0 or (w == 0 and not (dy > 0 or (dy == 0 and dx > 0))):
                        inside = False
                        break
                count[r, c] += inside
    return count, near


def _seg_dist(p, q, t):
    px, py = q[0] - p[0], q[1] - p[1]
    L2 = px * px + py * py
    u = min(1.0, max(0.0, ((t[0] - p[0]) * px + (t[1] - p[1]) * py) / L2))
    return math.hypot(p[0] + u * px - t[0], p[1] + u * py - t[1])
