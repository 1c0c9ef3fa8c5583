"""Files of OptimNetwork.save_debug (model/network.py:374-447): a binary PLY writer and the reference's arithmetic for
the debug images.  numpy and cv2 only: no trimesh, openmesh or pytorch3d on this path."""
import numpy as np
import torch


def write_ply(path, verts, faces):
    """Binary little-endian PLY of a triangle mesh: float32 x y z per vertex, an int32 triangle list per face.
    Vertices are written in the given order, unmerged (trimesh's export would merge duplicates and drop
    unreferenced ones)."""
    v = np.ascontiguousarray(torch.as_tensor(verts).detach().cpu().numpy(), dtype='<f4').reshape(-1, 3)
    f = np.ascontiguousarray(torch.as_tensor(faces).detach().cpu().numpy(), dtype='<i4').reshape(-1, 3)
    rows = np.empty(f.shape[0], dtype=[('n', 'u1'), ('v', '<i4', (3,))])
    rows['n'] = 3
    rows['v'] = f
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
              "property float z\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
              % (v.shape[0], f.shape[0]))
    with open(path, 'wb') as fh:
        fh.write(header.encode('ascii'))
        fh.write(v.tobytes())
        fh.write(rows.tobytes())


def mask_image(m):
    """(m * 255) truncated to uint8: the silhouette images m%d / mgm%d (network.py:390-398)."""
    return (m * 255.).detach().cpu().numpy().astype(np.uint8)


def color_image(colors, batch_inds, row_inds, col_inds, like):
    """rgb%d (network.py:426-430): white background, clamp((c/2+0.5)*255, 0, 255) at the covered pixels, truncated to
    uint8; channels in the order the network outputs them.  `like` is the [N,H,W,3] ground-truth image tensor."""
    tcolors = torch.clamp((colors / 2. + 0.5) * 255., min=0., max=255.)
    out = torch.ones_like(like) * 255.
    out[batch_inds, row_inds, col_inds, :] = tcolors
    return out.cpu().numpy().astype(np.uint8)


def normal_image(normals, batch_inds, row_inds, col_inds, like):
    """normal%d (network.py:432-436): white background, (n*0.5+0.5)*255 with channels [2,1,0], truncated to uint8."""
    tn = (normals * 0.5 + 0.5) * 255.
    out = torch.ones_like(like) * 255.
    out[batch_inds, row_inds, col_inds, :] = tn[:, [2, 1, 0]]
    return out.cpu().numpy().astype(np.uint8)


def gt_color_image(gtCs):
    """gtrgb%d (network.py:439): (gt/2+0.5)*255 truncated to uint8."""
    return ((gtCs / 2. + 0.5) * 255.).cpu().numpy().astype(np.uint8)
