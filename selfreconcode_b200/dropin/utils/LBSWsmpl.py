"""Skin-weight volume from a posed SMPL mesh (reference: utils/LBSWsmpl.py:1-52; one-time
initialiser, SURVEY.md section 8f-4).  For every voxel centre of the box: inverse-distance blend of the
skin weights of its `mean_neighbor` nearest SMPL vertices, then `smooth_times` damped 6-neighbour
smoothing passes with per-voxel renormalisation.  On CUDA float32 inputs with k and C up to 32 the blend runs on the
device kernels of csrc/lbsw_field.cu (exact difference norms, ties to the lower index), and so does the smoothing
when `smooth` is one of the two stock smoothers; other inputs take one cdist + top-k per chunk."""
import torch


def smooth_weights(weights, times=3):
    """weights [1,24,D,H,W]; returns the smoothed volume (entries < 5e-3 zeroed, LBSWsmpl.py:2-12)."""
    for _ in range(times):
        c = weights[:, :, 1:-1, 1:-1, 1:-1]
        mean = (weights[:, :, 2:, 1:-1, 1:-1] + weights[:, :, :-2, 1:-1, 1:-1] +
                weights[:, :, 1:-1, 2:, 1:-1] + weights[:, :, 1:-1, :-2, 1:-1] +
                weights[:, :, 1:-1, 1:-1, 2:] + weights[:, :, 1:-1, 1:-1, :-2]) / 6.0
        weights[:, :, 1:-1, 1:-1, 1:-1] = (c - mean) * 0.7 + mean
        weights = weights / weights.sum(1, keepdim=True)
    weights[weights < 5.e-3] = 0.0
    return weights


smooth_weights.lbsw_cut = 5.e-3     # the device smoother's final cut (0: model.Deformer's variant, no cut)


def voxel_centres(bmins, bmaxs, resolutions, device, align_corners=False):
    """World positions of the W*H*D lattice, x fastest (the [D,H,W] volume flattened)."""
    lo = torch.as_tensor(bmins, dtype=torch.float32, device=device).view(1, 3)
    hi = torch.as_tensor(bmaxs, dtype=torch.float32, device=device).view(1, 3)
    W, H, D = [int(r) for r in resolutions]
    res = torch.tensor([W, H, D], dtype=torch.float32, device=device).view(1, 3)
    z, y, x = torch.meshgrid(torch.arange(D, device=device), torch.arange(H, device=device),
                             torch.arange(W, device=device), indexing="ij")
    ijk = torch.stack([x, y, z], dim=0).reshape(3, -1).t().float()
    unit = ijk / (res - 1) if align_corners else ijk / res + (1.0 / res) / 2
    return unit * (hi - lo) + lo


def compute_lbswField(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners=False, mean_neighbor=5,
                      smooth_times=30, chunk=50000, smooth=smooth_weights):
    if (smpl_verts.is_cuda and smpl_verts.dtype == torch.float32 and smpl_ws.dtype == torch.float32
            and mean_neighbor <= 32 and smpl_ws.shape[-1] <= 32):
        from selfreconcode_b200 import ops
        field = ops.lbsw_field(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners, mean_neighbor)
        cut = getattr(smooth, "lbsw_cut", None)
        if cut is None:
            return smooth(field, smooth_times)
        return ops.lbsw_smooth(field, smooth_times, cut)
    W, H, D = [int(r) for r in resolutions]
    pts = voxel_centres(bmins, bmaxs, resolutions, smpl_verts.device, align_corners)
    out = []
    for part in torch.split(pts, chunk):
        dist, idx = torch.cdist(part, smpl_verts).topk(mean_neighbor, dim=-1, largest=False)
        w = 1. / dist.clamp(0.0001, 1.)
        w = w / w.sum(-1, keepdim=True)
        out.append((smpl_ws[idx.reshape(-1)] * w.reshape(-1, 1)).reshape(w.shape[0], mean_neighbor, -1).sum(1))
    field = torch.cat(out, dim=0).transpose(0, 1).reshape(1, -1, D, H, W)
    return smooth(field, smooth_times)
