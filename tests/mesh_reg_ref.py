"""Float64 restatement of pytorch3d 0.4.0's template mesh regularisers on one mesh, as OptimNetwork.computeTmpPcLoss
calls them (model/network.py:655-670), in pytorch3d's own terms: Meshes._compute_packed's hash unique for the edges,
Meshes.laplacian_packed's sparse L, mesh_edge_loss with target_length 0, and mesh_normal_consistency's three cross
products and literal pair comprehension with torch 1.10's cosine_similarity.  Gradients come from autograd.  pytorch3d
itself does not build against this project's torch, so this is the reference the kernels (csrc/mesh_reg.cu) are
checked against.

The negative-control switches restate rules that must NOT pass the same bars: `transpose` (L^T v in place of L v),
`half` (the edge loss over 2E) and `unique_pairs` (each unordered pair of an edge's faces once)."""
import torch

EPS = 1e-8


def packed_edges(faces, V):
    """Meshes._compute_packed: unique edges [E,2] (ascending V*a + b, a <= b) and face_to_edge [F,3] (column k = the
    edge opposite corner k)."""
    faces = torch.as_tensor(faces, dtype=torch.int64)
    F = faces.shape[0]
    v0, v1, v2 = faces.unbind(1)
    edges = torch.cat([torch.stack([v1, v2], 1), torch.stack([v2, v0], 1), torch.stack([v0, v1], 1)], 0)
    edges, _ = edges.sort(dim=1)
    uniq, inverse = torch.unique(V * edges[:, 0] + edges[:, 1], return_inverse=True)
    return torch.stack([uniq // V, uniq % V], 1), inverse.reshape(3, F).t().contiguous()


def laplacian_matrix(edges, V, transpose=False):
    """Meshes.laplacian_packed: A = both directions of every unique edge (duplicates summed), L = A / deg row-wise
    (0 for deg 0), minus I.  Sparse float64 [V,V] (built under no_grad, as pytorch3d does)."""
    with torch.no_grad():
        e0, e1 = edges[:, 0], edges[:, 1]
        idx = torch.cat([torch.stack([e0, e1], 1), torch.stack([e1, e0], 1)], 0).t()
        A = torch.sparse_coo_tensor(idx, torch.ones(idx.shape[1], dtype=torch.float64), (V, V)).coalesce()
        deg = torch.zeros(V, dtype=torch.float64).index_add_(0, A.indices()[0], A.values())
        inv = torch.where(deg > 0, 1.0 / deg.clamp(min=1e-300), deg)
        val = torch.cat([inv[e0], inv[e1]])
        diag = torch.arange(V).expand(2, V)
        idx = torch.cat([idx, diag], 1)
        val = torch.cat([val, -torch.ones(V, dtype=torch.float64)])
        if transpose:
            idx = idx.flip(0)
        return torch.sparse_coo_tensor(idx, val, (V, V)).coalesce()


def pair_table(faces, V, unique_pairs=False):
    """mesh_normal_consistency's bookkeeping: the (face, corner) entries sorted stably by edge, and the literal pairs
    [e[i], e[j]] for i in range(m-1) for j in range(1, m) if i != j over each edge's entries.
    -> (edge id per sorted entry, face row per sorted entry [3F,3], pairs [P,2] of sorted-entry indices)."""
    faces = torch.as_tensor(faces, dtype=torch.int64)
    F = faces.shape[0]
    edges, f2e = packed_edges(faces, V)
    edge_idx, order = f2e.reshape(3 * F).sort(stable=True)
    vert_idx = faces.view(1, F, 3).expand(3, F, 3).transpose(0, 1).reshape(3 * F, 3)[order]
    counts = edge_idx.bincount(minlength=edges.shape[0]).tolist()
    pairs, start = [], 0
    for m in counts:
        e = list(range(start, start + m))
        if unique_pairs:
            pairs += [[e[i], e[j]] for i in range(m) for j in range(i + 1, m)]
        else:
            pairs += [[e[i], e[j]] for i in range(m - 1) for j in range(1, m) if i != j]
        start += m
    return edge_idx, vert_idx, order, torch.tensor(pairs, dtype=torch.int64).reshape(-1, 2)


def topology(faces, V):
    """What the device topology holds: edges [E,2], face_to_edge [F,3] and the pairs as vertex ids [P,4] =
    (a, b, o_i, o_j), o = the entry's corner opposite the edge."""
    faces = torch.as_tensor(faces, dtype=torch.int64)
    edges, f2e = packed_edges(faces, V)
    edge_idx, vert_idx, order, pairs = pair_table(faces, V)
    corner = order % 3
    opp = vert_idx[torch.arange(vert_idx.shape[0]), corner]
    ab = edges[edge_idx[pairs[:, 0]]] if pairs.numel() else torch.zeros((0, 2), dtype=torch.int64)
    quads = torch.cat([ab, opp[pairs[:, 0]][:, None], opp[pairs[:, 1]][:, None]], 1) if pairs.numel() \
        else torch.zeros((0, 4), dtype=torch.int64)
    return dict(edges=edges, face_to_edge=f2e, pairs=quads, E=edges.shape[0], P=pairs.shape[0])


def laplacian_loss(verts, faces, transpose=False):
    """mesh_laplacian_smoothing(method='uniform'): sum_i |(L v)_i| / V."""
    V = verts.shape[0]
    edges, _ = packed_edges(faces, V)
    L = laplacian_matrix(edges, V, transpose)
    return torch.sparse.mm(L, verts).norm(dim=1).sum() / V


def edge_loss(verts, faces, half=False):
    """mesh_edge_loss(target_length=0.): sum_e (|v_a - v_b| - 0)^2 / E."""
    edges, _ = packed_edges(faces, verts.shape[0])
    v0, v1 = verts[edges].unbind(1)
    loss = ((v0 - v1).norm(dim=1, p=2) - 0.0) ** 2.0
    return loss.sum() / (2 * edges.shape[0] if half else edges.shape[0])


def cosine_similarity_110(x1, x2, eps=EPS):
    """torch 1.10's cosine_similarity: w12 / sqrt(clamp_min(w1 * w2, eps^2))."""
    w12 = (x1 * x2).sum(1)
    w1, w2 = (x1 * x1).sum(1), (x2 * x2).sum(1)
    return w12 / (w1 * w2).clamp_min(eps * eps).sqrt()


def normal_consistency(verts, faces, unique_pairs=False):
    """mesh_normal_consistency: the three cross products of every (face, corner) entry against its edge, then
    1 - cos(n_i, -n_j) over the pairs, averaged (0 without pairs).  An entry whose normal is zero for every vertex
    position (its corner on the edge, or a self-edge: faces with a repeated index) gets an exact 0, so such a pair
    contributes 1 - 0 and no gradient.  Computed literally, rounding leaves ~1e-17 there, which the eps clamp's 1/eps
    turns into gradients of order 1e-8 |n_i| / eps with no meaning."""
    V = verts.shape[0]
    edges, _ = packed_edges(faces, V)
    edge_idx, vert_idx, _, pairs = pair_table(faces, V, unique_pairs)
    if pairs.shape[0] == 0:
        return verts.sum() * 0.0
    a, b = edges[edge_idx, 0], edges[edge_idx, 1]
    v0, v1 = verts[a], verts[b]
    n = 0.0
    for c in range(3):
        # the products pytorch3d notes are zero (a corner on the edge, or a self-edge) are taken as exact zeros
        live = ((vert_idx[:, c] != a) & (vert_idx[:, c] != b) & (a != b)).to(verts.dtype)[:, None]
        n = n + torch.linalg.cross(v1 - v0, verts[vert_idx[:, c]] - v0, dim=1) * live
    loss = 1 - cosine_similarity_110(n[pairs[:, 0]], -n[pairs[:, 1]])
    return loss.sum() / pairs.shape[0]


def regularizers(verts, faces, **controls):
    """[3] = (laplacian, edge, normal consistency), float64, differentiable w.r.t. verts."""
    v = verts.double()
    return torch.stack([laplacian_loss(v, faces, controls.get("transpose", False)),
                        edge_loss(v, faces, controls.get("half", False)),
                        normal_consistency(v, faces, controls.get("unique_pairs", False))])


def values_and_grads(verts, faces, cot=(1.0, 1.0, 1.0), **controls):
    """(values [3], d(cot . values)/dverts [V,3]) in float64."""
    v = torch.as_tensor(verts, dtype=torch.float64).detach().clone().requires_grad_(True)
    r = regularizers(v, faces, **controls)
    g, = torch.autograd.grad((r * torch.as_tensor(cot, dtype=torch.float64)).sum(), [v])
    return r.detach(), g
