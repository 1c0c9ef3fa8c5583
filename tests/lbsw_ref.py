"""float64 restatement of the skin-weight volume (the reference's compute_lbswField / smooth_weights,
model/Deformer.py:235-284, utils/LBSWsmpl.py:2-52) that the device kernels of csrc/lbsw_field.cu are checked against.

Neighbours come from exact difference norms (not cdist's |x|^2 + |y|^2 - 2 x.y) and are ordered by (d, vertex index);
the blend and the passes run in float64.  Works on CPU or CUDA tensors.  The knobs of `centres` (`offset`) and
`smooth` (`in_place`, `renorm`, `cut_every_pass`) exist for the negative controls of test_lbsw_ref_cpu.py."""
import torch


def centres(bmins, bmaxs, resolutions, align_corners=False, offset=0.0, device="cpu"):
    """Voxel centres [W*H*D,3] (x fastest) in float64; `offset` shifts them by that many voxels on every axis."""
    W, H, D = [int(r) for r in resolutions]
    lo = torch.as_tensor(bmins, dtype=torch.float64, device=device).view(1, 3)
    hi = torch.as_tensor(bmaxs, dtype=torch.float64, device=device).view(1, 3)
    res = torch.tensor([W, H, D], dtype=torch.float64, device=device).view(1, 3)
    z, y, x = torch.meshgrid(torch.arange(D, device=device), torch.arange(H, device=device),
                             torch.arange(W, device=device), indexing="ij")
    ijk = torch.stack([x, y, z], dim=0).reshape(3, -1).t().double() + offset
    unit = ijk / (res - 1) if align_corners else (ijk + 0.5) / res
    return unit * (hi - lo) + lo


def knn(pts, verts, k, chunk=20000):
    """(d [N,k+1], idx [N,k+1]): the k+1 nearest vertices of every point by exact float64 difference norms, ordered
    by (d, index) (a stable sort over the index-ordered candidates).  The (k+1)-th is returned for tie checks."""
    verts = verts.double()
    kk = min(k + 1, verts.shape[0])
    ds, ids = [], []
    for part in torch.split(pts.double(), chunk):
        d = (part[:, None, :] - verts[None, :, :]).norm(dim=-1)
        d, i = torch.sort(d, dim=1, stable=True)
        ds.append(d[:, :kk].clone())
        ids.append(i[:, :kk].clone())
    return torch.cat(ds), torch.cat(ids)


def blend(d, idx, vert_ws, k, chunk=100000):
    """[N,C]: inverse-distance weights 1 / min(max(d, 1e-4), 1), normalised, over the first k neighbours."""
    out = []
    for dd, ii in zip(torch.split(d, chunk), torch.split(idx, chunk)):
        w = 1.0 / dd[:, :k].clamp(1e-4, 1.0)
        w = w / w.sum(-1, keepdim=True)
        out.append((vert_ws.double()[ii[:, :k]] * w.unsqueeze(-1)).sum(1))
    return torch.cat(out)


def field(bmins, bmaxs, resolutions, verts, vert_ws, k, align_corners=False, pts=None, offset=0.0):
    """[1,C,D,H,W] float64 blend and the (k+1)-NN distances [N,k+1]; `pts` overrides the centres."""
    W, H, D = [int(r) for r in resolutions]
    if pts is None:
        pts = centres(bmins, bmaxs, resolutions, align_corners, offset, verts.device)
    d, idx = knn(pts, verts, k)
    f = blend(d, idx, vert_ws, k)
    return f.t().reshape(1, -1, D, H, W), d


def smooth(field, times, cut=0.0, in_place=False, renorm=True, cut_every_pass=False):
    """`times` damped 6-neighbour passes over [1,C,D,H,W] (float64): interior c -> (c - mean) * 0.7 + mean with mean
    from the previous volume (Jacobi), then division by the channel sum; values below `cut` zeroed after the last pass
    (after the blend when times == 0).  in_place = Gauss-Seidel order (each voxel sees its already-updated
    neighbours), a negative control."""
    w = field.double().clone()
    for t in range(times):
        if in_place:
            _, _, D, H, W = w.shape
            for z in range(1, D - 1):
                for y in range(1, H - 1):
                    for x in range(1, W - 1):
                        m = (w[0, :, z + 1, y, x] + w[0, :, z - 1, y, x] + w[0, :, z, y + 1, x] +
                             w[0, :, z, y - 1, x] + w[0, :, z, y, x + 1] + w[0, :, z, y, x - 1]) / 6.0
                        w[0, :, z, y, x] = (w[0, :, z, y, x] - m) * 0.7 + m
        else:
            new = w.clone()
            c = w[:, :, 1:-1, 1:-1, 1:-1]
            mean = (w[:, :, 2:, 1:-1, 1:-1] + w[:, :, :-2, 1:-1, 1:-1] + w[:, :, 1:-1, 2:, 1:-1] +
                    w[:, :, 1:-1, :-2, 1:-1] + w[:, :, 1:-1, 1:-1, 2:] + w[:, :, 1:-1, 1:-1, :-2]) / 6.0
            new[:, :, 1:-1, 1:-1, 1:-1] = (c - mean) * 0.7 + mean
            w = new
        if renorm:
            w = w / w.sum(1, keepdim=True)
        if cut > 0 and cut_every_pass and t < times - 1:
            w = torch.where(w < cut, torch.zeros_like(w), w)
    if cut > 0:
        w = torch.where(w < cut, torch.zeros_like(w), w)
    return w
