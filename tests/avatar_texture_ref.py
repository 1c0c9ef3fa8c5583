"""Float64 restatement of the textured avatar's rules (csrc/avatar_texture.cu, selfreconcode_b200.avatar): the
coverage-weighted mip pyramid, the UV interpolation, the analytic screen-space footprint, trilinear sampling, and the
linear blend skinning of the exported avatar."""
import numpy as np


def mip_sizes(Ht, Wt):
    out = [(Ht, Wt)]
    while Ht > 1 or Wt > 1:
        Ht, Wt = (Ht + 1) // 2, (Wt + 1) // 2
        out.append((Ht, Wt))
    return out


def mips(texture_u8, coverage):
    """[Ht,Wt,3] uint8, [Ht,Wt] -> list of [H_l,W_l,4] float64 levels (r, g, b, w)."""
    t = np.asarray(texture_u8, np.float64) / 255.
    lv = [np.concatenate([t, (np.asarray(coverage) != 0)[..., None].astype(np.float64)], -1)]
    for Hd, Wd in mip_sizes(*t.shape[:2])[1:]:
        p = lv[-1]
        Hs, Ws = p.shape[:2]
        pad = np.zeros((2 * Hd, 2 * Wd, 4))
        valid = np.zeros((2 * Hd, 2 * Wd))
        pad[:Hs, :Ws], valid[:Hs, :Ws] = p, 1.
        blocks = pad.reshape(Hd, 2, Wd, 2, 4)
        vb = valid.reshape(Hd, 2, Wd, 2)
        cnt = vb.sum((1, 3))
        w = blocks[..., 3]
        sw = w.sum((1, 3))
        swc = (blocks[..., :3] * w[..., None]).sum((1, 3))
        plain = blocks[..., :3].sum((1, 3)) / cnt[..., None]
        with np.errstate(invalid="ignore", divide="ignore"):
            col = np.where(sw[..., None] > 0, swc / sw[..., None], plain)
        lv.append(np.concatenate([col, (sw / cnt)[..., None]], -1))
    return lv


def bilinear(level, x, y):
    """level [H,W,C] at texel coordinates x, y (arrays), clamp-to-edge -> [..., C]."""
    Hl, Wl = level.shape[:2]
    x, y = np.clip(x, -1., Wl), np.clip(y, -1., Hl)
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = (x - x0)[..., None], (y - y0)[..., None]
    c0, c1 = np.clip(x0, 0, Wl - 1).astype(np.int64), np.clip(x0 + 1, 0, Wl - 1).astype(np.int64)
    r0, r1 = np.clip(y0, 0, Hl - 1).astype(np.int64), np.clip(y0 + 1, 0, Hl - 1).astype(np.int64)
    return (1 - fy) * ((1 - fx) * level[r0, c0] + fx * level[r0, c1]) + fy * ((1 - fx) * level[r1, c0] + fx * level[r1, c1])


def sample(levels, u, v, lam):
    """Trilinear lookup of the pyramid at uv with level parameter lam (already clamped to [0, L-1]) -> [..., 3]."""
    L = len(levels)
    l0 = np.floor(lam).astype(np.int64)
    fr = (lam - l0)[..., None]
    l1 = np.minimum(l0 + 1, L - 1)
    out = np.zeros(np.shape(u) + (3,))
    for l in range(L):
        Hl, Wl = levels[l].shape[:2]
        c = bilinear(levels[l][..., :3], u * Wl - 0.5, (1. - v) * Hl - 0.5)
        out += np.where((l0 == l)[..., None], (1. - fr) * c, 0.) + np.where((l1 == l)[..., None], fr * c, 0.)
    return out


def footprint(xy, iz, uv, px, py, Ht, Wt):
    """Analytic footprint of a face's UV map at pixel centres (px, py).  xy [...,3,2] screen corners, iz [...,3] =
    1 / Z, uv [...,3,2] -> rho in level-0 texels (the larger length of d(u Wt, v Ht)/dcol and /drow)."""
    x, y = xy[..., 0], xy[..., 1]
    ia = 1. / ((x[..., 1] - x[..., 0]) * (y[..., 2] - y[..., 0]) - (x[..., 2] - x[..., 0]) * (y[..., 1] - y[..., 0]))
    la = np.stack([(x[..., 1] - px) * (y[..., 2] - py) - (x[..., 2] - px) * (y[..., 1] - py),
                   (x[..., 2] - px) * (y[..., 0] - py) - (x[..., 0] - px) * (y[..., 2] - py),
                   (x[..., 0] - px) * (y[..., 1] - py) - (x[..., 1] - px) * (y[..., 0] - py)], -1) * ia[..., None]
    ldx = np.stack([y[..., 1] - y[..., 2], y[..., 2] - y[..., 0], y[..., 0] - y[..., 1]], -1) * ia[..., None]
    ldy = np.stack([x[..., 2] - x[..., 1], x[..., 0] - x[..., 2], x[..., 1] - x[..., 0]], -1) * ia[..., None]
    q = la * iz
    S = q.sum(-1, keepdims=True)
    b = q / S
    bx = (ldx * iz - b * (ldx * iz).sum(-1, keepdims=True)) / S
    by = (ldy * iz - b * (ldy * iz).sum(-1, keepdims=True)) / S
    scale = np.array([Wt, Ht], np.float64)
    gx = (bx[..., None] * uv).sum(-2) * scale
    gy = (by[..., None] * uv).sum(-2) * scale
    return np.maximum(np.linalg.norm(gx, axis=-1), np.linalg.norm(gy, axis=-1))


def level_param(rho, L):
    with np.errstate(divide="ignore", invalid="ignore"):
        lam = np.log2(rho)
    return np.clip(np.nan_to_num(lam, nan=0., neginf=0.), 0., L - 1)


def shade(p2f, bary, verts_screen, faces, ft, vt, levels, background, flip_v=True, texel_shift=0.):
    """The shader on given fragments: p2f [N,H,W] packed ids, bary [N,H,W,3], verts_screen [N,V,3] -> [N,H,W,4].
    background = 3 floats or [N,H,W,3] uint8.  flip_v / texel_shift change the UV convention (negative controls)."""
    p2f = np.asarray(p2f)
    N, H, W = p2f.shape
    F = faces.shape[0]
    out = np.zeros((N, H, W, 4))
    if np.ndim(background) == 1:
        out[..., :3] = np.asarray(background, np.float64)
    else:
        out[..., :3] = np.asarray(background, np.float64) / 255.
    cov = p2f >= 0
    n_i, r_i, c_i = np.nonzero(cov)
    pf = p2f[cov]
    m, f = pf // F, pf % F
    vs = np.asarray(verts_screen, np.float64)
    corners = vs[m[:, None], faces[f]]                        # [P,3,3]
    uvc = np.asarray(vt, np.float64)[ft[f]]                   # [P,3,2]
    b = np.asarray(bary, np.float64)[cov]
    u, v = (b * uvc[..., 0]).sum(-1), (b * uvc[..., 1]).sum(-1)
    Ht, Wt = levels[0].shape[:2]
    rho = footprint(corners[..., :2], 1. / corners[..., 2], uvc, c_i.astype(np.float64), r_i.astype(np.float64), Ht, Wt)
    lam = level_param(rho, len(levels))
    if not flip_v:
        v = 1. - v
    out[cov, :3] = sample(levels, u + texel_shift / Wt, v - texel_shift / Ht, lam)
    out[cov, 3] = 1.
    return out, lam


# ---- linear blend skinning of an exported avatar ------------------------------------------------------------------
def rodrigues(theta):
    """[...,3] axis-angle -> [...,3,3] (the skinner's rule: angle of theta + 1e-8)."""
    theta = np.asarray(theta, np.float64)
    angle = np.linalg.norm(theta + 1e-8, axis=-1, keepdims=True)
    k = theta / angle
    half = angle[..., 0] * 0.5
    w, (x, y, z) = np.cos(half), np.moveaxis(np.sin(half)[..., None] * k, -1, 0)
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (w * y + x * z),
                     2 * (w * z + x * y), w * w - x * x + y * y - z * z, 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (w * x + y * z), w * w - x * x - y * y + z * z], -1).reshape(
        theta.shape[:-1] + (3, 3))


def bone_chain(poses, Js, parents):
    """poses [T,24,3], Js [24,3], parents [24] -> G [T,24,4,4]: G_0 = [R_0, Js_0], G_j = G_parent [R_j, Js_j - Js_p]."""
    poses = np.asarray(poses, np.float64).reshape(-1, 24, 3)
    Js = np.asarray(Js, np.float64)
    R = rodrigues(poses)
    T = poses.shape[0]
    G = np.zeros((T, 24, 4, 4))
    for j in range(24):
        A = np.zeros((T, 4, 4))
        A[:, :3, :3] = R[:, j]
        A[:, 3, 3] = 1.
        A[:, :3, 3] = Js[j] - (Js[int(parents[j])] if j > 0 else 0.)
        G[:, j] = A if j == 0 else G[:, int(parents[j])] @ A
    return G


def lbs(avatar, poses, trans):
    """Posed vertices [T,V,3] of an export_avatar .npz (dict-like) for poses [T,24,3] / [T,72], trans [T,3]."""
    G = bone_chain(poses, avatar["Js"], avatar["parents"])
    A = G @ np.asarray(avatar["init_pose"], np.float64)[None]
    w = np.asarray(avatar["skin_weights"], np.float64)
    M = np.einsum("vj,tjab->tvab", w, A)
    v = np.asarray(avatar["verts"], np.float64)
    return np.einsum("tvab,vb->tva", M[..., :3, :3], v) + M[..., :3, 3] + np.asarray(trans, np.float64).reshape(-1, 1, 3)
