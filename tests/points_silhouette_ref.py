"""Float64 numpy restatement of the soft point-cloud silhouette of the optimisation step (model/network.py:495-505):
pytorch3d 0.4.0's PointsRasterizer (points_per_pixel K, radius r) + AlphaCompositor(background_color=None), unit
features, written in pytorch3d's own terms, with its analytic gradient.  The reference for csrc/points_silhouette.cu.

  projection  view = p R + T; NDC = K-matrix transform of view (RectifiedPerspectiveCameras: the screen-space camera
              converted by _get_sfm_calibration_matrix with image_size), NDC z replaced by the view-space Z
              (PointsRasterizer.transform).
  pixels      pixel (i, j) of the output is NDC (PixToNdc(W-1-j, W), PixToNdc(H-1-i, H)), PixToNdc(t, S) = -1 +
              (2t+1)/S: each axis spans [-1, 1] on its own, so pixels are anisotropic in NDC on non-square images.
              This is the 0.4.0 convention RectifiedPerspectiveCameras is written for; later pytorch3d releases
              scale the shorter side to [-1, 1] instead.  Square images are the same under both.
  coverage    Z >= 0 and d2 = |NDC_p - NDC_pixel|^2 < r^2 (strict, CheckPixelInsidePoint).
  selection   per pixel the K covering points of smallest Z, equal Z by index (the rasteriser visits points in
              index order and replaces only on a strictly smaller Z).
  compositing w = 1 - d2 / r^2; mask = sum_k w_k prod_{j<k} (1 - w_j) in the kept order (the k-loop of
              AlphaCompositor with features 1).
  gradient    through d2 only: dmask/dw_p = prod_{q != p} (1 - w_q); dd2/dNDC_p = 2 (NDC_p - NDC_pixel).
"""
import numpy as np


def pix_to_ndc(t, S):
    return -1.0 + (2.0 * t + 1.0) / S


def calibration_ndc(focal, pp, H, W):
    """_get_sfm_calibration_matrix(image_size=(W, H)) for one camera: 4x4 K in NDC."""
    fx, fy = focal[0] / (W / 2.0), focal[1] / (H / 2.0)
    px, py = 1.0 - 1.0 / W - pp[0] / (W / 2.0), 1.0 - 1.0 / H - pp[1] / (H / 2.0)
    K = np.zeros((4, 4))
    K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[3, 2], K[2, 3] = fx, fy, px, py, 1.0, 1.0
    return K


def project_ndc(verts, R, T, focal, pp, H, W):
    """verts [N,V,3], camera n for frame n -> NDC (x, y, view Z) [N,V,3] in float64."""
    out = []
    for n in range(verts.shape[0]):
        view = verts[n].astype(np.float64) @ R[n].astype(np.float64) + T[n].astype(np.float64)
        h = np.concatenate([view, np.ones((view.shape[0], 1))], 1) @ calibration_ndc(focal[n], pp[n], H, W).T
        out.append(np.stack([h[:, 0] / h[:, 3], h[:, 1] / h[:, 3], view[:, 2]], 1))
    return np.stack(out)


def screen_to_ndc(pts_screen, H, W):
    """(col, row, Z) of the built-in projection -> (NDC x, NDC y, Z): col is the pixel coordinate whose centre is
    PixToNdc(W-1-col, W)."""
    p = np.asarray(pts_screen, np.float64)
    return np.stack([pix_to_ndc(W - 1 - p[..., 0], W), pix_to_ndc(H - 1 - p[..., 1], H), p[..., 2]], -1)


def _pairs(ndc, H, W, r, isotropic):
    """Every (frame, point, pixel) with d2 < r^2 and Z >= 0, with its d2 and NDC offsets.  Only pixels within r of
    the point along each axis are examined (a farther pixel cannot be covered)."""
    N, V, _ = ndc.shape
    sx, sy = (2.0 / min(H, W),) * 2 if isotropic else (2.0 / W, 2.0 / H)
    out = []
    for n in range(N):
        x, y, z = ndc[n, :, 0], ndc[n, :, 1], ndc[n, :, 2]
        ok = (z >= 0) & np.isfinite(x) & np.isfinite(y)
        # pixel coordinate of the point (inverse of PixToNdc with the flip)
        cj = W - 1 - ((x + 1.0) * W - 1.0) / 2.0
        ci = H - 1 - ((y + 1.0) * H - 1.0) / 2.0
        ex, ey = int(np.ceil(r / sx)) + 1, int(np.ceil(r / sy)) + 1
        pid = np.nonzero(ok)[0]
        for dj in range(-ex, ex + 1):
            for di in range(-ey, ey + 1):
                j = np.round(cj[pid]).astype(np.int64) + dj
                i = np.round(ci[pid]).astype(np.int64) + di
                inside = (j >= 0) & (j < W) & (i >= 0) & (i < H)
                p, j, i = pid[inside], j[inside], i[inside]
                if isotropic:   # pixel centres 2/min(H,W) apart on both axes, about the image centre
                    xp, yp = -(j - (W - 1) / 2.0) * sx, -(i - (H - 1) / 2.0) * sy
                    xq, yq = -(cj[p] - (W - 1) / 2.0) * sx, -(ci[p] - (H - 1) / 2.0) * sy
                else:
                    xp, yp = pix_to_ndc(W - 1 - j, W), pix_to_ndc(H - 1 - i, H)
                    xq, yq = x[p], y[p]
                dx, dy = xq - xp, yq - yp
                d2 = dx * dx + dy * dy
                c = d2 < r * r
                out.append((np.full(c.sum(), n), p[c], i[c], j[c], d2[c], dx[c], dy[c], z[p[c]]))
    cat = [np.concatenate([o[k] for o in out]) if out else np.zeros(0) for k in range(8)]
    return dict(n=cat[0].astype(np.int64), p=cat[1].astype(np.int64), i=cat[2].astype(np.int64),
                j=cat[3].astype(np.int64), d2=cat[4], dx=cat[5], dy=cat[6], z=cat[7])


def rasterize(ndc, H, W, r, K, isotropic=False):
    """Kept (pixel, point) pairs in per-pixel (Z, index) order with their slot k: dict of arrays + `pix` (flat
    n*H*W + i*W + j) and `n_cover` (covering points per pixel, before truncation to K)."""
    P = _pairs(ndc, H, W, r, isotropic)
    pix = (P["n"] * H + P["i"]) * W + P["j"]
    order = np.lexsort((P["p"], P["z"], pix))
    P = {k: v[order] for k, v in P.items()}
    pix = pix[order]
    start = np.r_[0, np.nonzero(np.diff(pix))[0] + 1] if pix.size else np.zeros(0, np.int64)
    first = np.zeros(pix.size, np.int64)
    first[start] = start
    first = np.maximum.accumulate(first) if pix.size else first
    slot = np.arange(pix.size) - first
    n_cover = np.bincount(pix, minlength=ndc.shape[0] * H * W)
    keep = slot < K if K is not None else np.ones(pix.size, bool)
    P = {k: v[keep] for k, v in P.items()}
    P["pix"], P["slot"], P["n_cover"] = pix[keep], slot[keep], n_cover
    return P


def composite(P, N, H, W, r, r2_scale=True):
    """AlphaCompositor k-loop with unit features -> mask [N,H,W]; also the per-pair weight w.  r2_scale=False drops
    the 1/r^2 of the weight (a negative control)."""
    w = 1.0 - (P["d2"] / (r * r) if r2_scale else P["d2"])
    acc = np.zeros(N * H * W)
    T = np.ones(N * H * W)
    for k in range(int(P["slot"].max()) + 1 if P["slot"].size else 0):
        s = P["slot"] == k
        acc[P["pix"][s]] += w[s] * T[P["pix"][s]]
        T[P["pix"][s]] *= 1.0 - w[s]
    return acc.reshape(N, H, W), w


def silhouette(ndc, H, W, r, K, isotropic=False, r2_scale=True):
    P = rasterize(ndc, H, W, r, K, isotropic)
    return composite(P, ndc.shape[0], H, W, r, r2_scale)[0]


def silhouette_grad(ndc, H, W, r, K, grad_mask, with_others=True):
    """dL/d(NDC x, NDC y) [N,V,2] for L = sum grad_mask * mask: dmask/dw_p = prod_{q != p}(1 - w_q) from prefix and
    suffix products over the pixel's kept points (no division: exact with w = 1 factors)."""
    N, V = ndc.shape[0], ndc.shape[1]
    P = rasterize(ndc, H, W, r, K)
    _, w = composite(P, N, H, W, r)
    om = 1.0 - w
    kmax = int(P["slot"].max()) + 1 if P["slot"].size else 0
    pre = np.ones(om.size)
    T = np.ones(N * H * W)
    for k in range(kmax):
        s = P["slot"] == k
        pre[s] = T[P["pix"][s]]
        T[P["pix"][s]] *= om[s]
    suf = np.ones(om.size)
    T = np.ones(N * H * W)
    for k in range(kmax - 1, -1, -1):
        s = P["slot"] == k
        suf[s] = T[P["pix"][s]]
        T[P["pix"][s]] *= om[s]
    others = pre * suf if with_others else np.ones(om.size)
    g = grad_mask.reshape(-1)[P["pix"]] * others * (-1.0 / (r * r))     # dL/dd2
    out = np.zeros((N, V, 2))
    np.add.at(out, (P["n"], P["p"], 0), g * 2.0 * P["dx"])
    np.add.at(out, (P["n"], P["p"], 1), g * 2.0 * P["dy"])
    return out


def ndc_grad_to_screen(g_ndc, H, W):
    """dL/d(col, row, Z) from dL/d(NDC x, NDC y): x = 1 - (2 col + 1)/W, y = 1 - (2 row + 1)/H."""
    return np.concatenate([g_ndc[..., :1] * (-2.0 / W), g_ndc[..., 1:2] * (-2.0 / H),
                           np.zeros(g_ndc.shape[:-1] + (1,))], -1)


def borderline_points(ndc, H, W, r, K, rel=1e-6):
    """[N,V] bool: points within rounding of a decision -- |d2 - r^2| <= rel r^2 at some pixel, or a depth equal to
    that of the K-th kept point of a pixel with more than K covering points (other than being that point)."""
    N, V = ndc.shape[0], ndc.shape[1]
    out = np.zeros((N, V), bool)
    P = _pairs(ndc, H, W, r * (1.0 + rel), False)
    near = np.abs(P["d2"] - r * r) <= rel * r * r
    out[P["n"][near], P["p"][near]] = True
    R = rasterize(ndc, H, W, r, None)
    crowded = R["n_cover"][R["pix"]] > K
    kth = crowded & (R["slot"] == K - 1)
    zk = np.full(N * H * W, np.nan)
    zk[R["pix"][kth]] = R["z"][kth]
    tie = crowded & (R["z"] == zk[R["pix"]]) & (R["slot"] != K - 1)
    out[R["n"][tie], R["p"][tie]] = True
    return out
