"""Float64 numpy restatement of the texture-atlas rule of selfreconcode_b200.texture (the reference's
texture_mesh_extract.py:57-144 and texture_mesh_prepare.py:81; DESIGN.md section 3.3).

UV raster: texel (i, j) is the pixel centre (col j, row i) of the screen vertices (u R - 0.5, (1 - v) R - 0.5); a texel
belongs to the lowest-numbered non-degenerate UV face whose closed triangle contains it (all faces are at depth 1, so
the rasteriser's (depth, face) key picks the lowest face id).  Accumulation: per frame, alpha = sum b_i a_v over a usable
face (0 otherwise); alpha > min slot alpha overwrites the first slot holding that minimum with (bilinear(image, sum b_i
s_v) / 255, alpha, frame id).  Finish: count of slots above c0, mask_final = count >= min_views, np.nanmedian of the
filled slots, view id of the first largest alpha."""
import numpy as np


def frame_ids(num, frame_num):
    if num < 1 or num > frame_num:
        raise ValueError("num must lie in [1, frame_num]")
    return np.ceil(np.arange(num) * frame_num * 1. / num).astype(np.int64)


def uv_screen(vt, R):
    """The atlas screen vertices in float32 arithmetic (as the baker forms them), returned as float64."""
    vt = np.asarray(vt, np.float32)
    R32 = np.float32(R)
    x = vt[:, 0] * R32 - np.float32(0.5)
    y = (np.float32(1.) - vt[:, 1]) * R32 - np.float32(0.5)
    return np.stack([x, y], 1).astype(np.float64)


def uv_raster(xy, ft, R, edge_eps=1e-6):
    """-> (face [R,R] int64 (-1 = none), bary [R,R,3] float64, near_edge [R,R] bool, overlap [R,R] bool).  near_edge
    marks texels whose smallest barycentric in some face lies within edge_eps of 0 (decided differently by any two
    roundings); overlap marks texels strictly inside two or more faces (an atlas whose faces overlap: the rasteriser's
    depth 1 / (l0 + l1 + l2) carries a rounding there, so any of those faces may take the texel)."""
    xy = np.asarray(xy, np.float64)
    ft = np.asarray(ft, np.int64)
    face = -np.ones((R, R), np.int64)
    bary = np.zeros((R, R, 3))
    near = np.zeros((R, R), bool)
    inside = np.zeros((R, R), np.int32)
    for k, (a, b, c) in enumerate(ft):
        x0, y0 = xy[a]
        x1, y1 = xy[b]
        x2, y2 = xy[c]
        area = (x1 - x0) * (y2 - y0) - (x2 - x0) * (y1 - y0)
        if abs(area) < 1e-12:
            continue
        c0, c1 = max(0, int(np.ceil(min(x0, x1, x2)))), min(R - 1, int(np.floor(max(x0, x1, x2))))
        r0, r1 = max(0, int(np.ceil(min(y0, y1, y2)))), min(R - 1, int(np.floor(max(y0, y1, y2))))
        if c1 < c0 or r1 < r0:
            continue
        py, px = np.meshgrid(np.arange(r0, r1 + 1, dtype=np.float64), np.arange(c0, c1 + 1, dtype=np.float64),
                             indexing="ij")
        l0 = ((x1 - px) * (y2 - py) - (x2 - px) * (y1 - py)) / area
        l1 = ((x2 - px) * (y0 - py) - (x0 - px) * (y2 - py)) / area
        l2 = ((x0 - px) * (y1 - py) - (x1 - px) * (y0 - py)) / area
        lm = np.minimum(np.minimum(l0, l1), l2)
        near[r0:r1 + 1, c0:c1 + 1] |= np.abs(lm) <= edge_eps
        inside[r0:r1 + 1, c0:c1 + 1] += lm > edge_eps
        take = (lm >= 0) & (face[r0:r1 + 1, c0:c1 + 1] < 0)
        sub_f = face[r0:r1 + 1, c0:c1 + 1]
        sub_b = bary[r0:r1 + 1, c0:c1 + 1]
        sub_f[take] = k
        sub_b[take] = np.stack([l0, l1, l2], -1)[take]
    return face, bary, near, inside >= 2


def bilinear(image, p):
    """image [H,W,C], p [...,2] = (col, row) with pixel centres at integers, clamp-to-edge -> [..., C] float64."""
    img = np.asarray(image, np.float64)
    H, W = img.shape[:2]
    x = np.clip(p[..., 0], -1., W)
    y = np.clip(p[..., 1], -1., H)
    fx0, fy0 = np.floor(x), np.floor(y)
    fx, fy = (x - fx0)[..., None], (y - fy0)[..., None]
    x0 = np.clip(fx0, 0, W - 1).astype(np.int64)
    x1 = np.clip(fx0 + 1, 0, W - 1).astype(np.int64)
    y0 = np.clip(fy0, 0, H - 1).astype(np.int64)
    y1 = np.clip(fy0 + 1, 0, H - 1).astype(np.int64)
    top = (1 - fx) * img[y0, x0] + fx * img[y0, x1]
    bot = (1 - fx) * img[y1, x0] + fx * img[y1, x1]
    return (1 - fy) * top + fy * bot


class Slots:
    """The reference's tex_agg / normal_agg / viewid_agg over T texels, slot-first; `close` marks texels on which a
    comparison came within `tol` (an update test, the first-minimum pick, or the first-maximum pick at finish)."""

    def __init__(self, T, S, c0, tol=1e-6):
        self.rgb = np.full((S, T, 3), np.nan)
        self.alpha = np.full((S, T), float(c0))
        self.view = -np.ones((S, T), np.int64)
        self.c0, self.tol = float(c0), tol
        self.close = np.zeros(T, bool)

    def update(self, alpha, colour_fn, frame_id):
        """alpha [T] of this frame; colour_fn(mask) -> [n,3] colours of the texels that take a slot."""
        T = alpha.shape[0]
        srt = np.sort(self.alpha, 0)
        mn = srt[0]
        arg = np.argmin(self.alpha, 0)          # first minimum
        upd = alpha > mn
        self.close |= (alpha > 0) & (np.abs(alpha - mn) <= self.tol)
        if self.alpha.shape[0] > 1:
            self.close |= upd & (srt[1] - mn <= self.tol) & (srt[1] > self.c0)
        t = np.nonzero(upd)[0]
        if t.size:
            self.rgb[arg[t], t] = colour_fn(upd)
            self.alpha[arg[t], t] = alpha[t]
            self.view[arg[t], t] = frame_id
        return upd


def accumulate(slots, texel_face, texel_bary, screen, faces, weight, usable, image, frame_id):
    """One frame (texture_mesh_extract.py:101-123) on given per-vertex / per-face inputs."""
    k = np.asarray(texel_face, np.int64)
    b = np.asarray(texel_bary, np.float64)
    fv = np.asarray(faces, np.int64)[k]                              # [T,3]
    ok = np.asarray(usable)[k] > 0
    alpha = (b * np.asarray(weight, np.float64)[fv]).sum(1)
    alpha[~ok] = 0.
    s = np.asarray(screen, np.float64)[:, :2]

    def colour(m):
        p = (b[m][:, :, None] * s[fv[m]]).sum(1)
        return bilinear(image, p) / 255.
    return slots.update(alpha, colour, frame_id)


def finish(slots, min_views):
    """-> (tex_median [T,3], mask_final [T], view_id [T], count [T]) (texture_mesh_extract.py:131-144)."""
    filled = slots.alpha > slots.c0
    count = filled.sum(0)
    mask_final = count >= min_views
    rgb = np.where(filled[..., None], slots.rgb, np.nan)
    med = np.zeros((rgb.shape[1], 3))
    if mask_final.any():
        med[mask_final] = np.nanmedian(rgb[:, mask_final], axis=0)
    srt = np.sort(slots.alpha, 0)
    if slots.alpha.shape[0] > 1:
        slots.close |= mask_final & (srt[-1] - srt[-2] <= slots.tol)
    view = slots.view[np.argmax(slots.alpha, 0), np.arange(slots.alpha.shape[1])]
    view[~mask_final] = -1
    return med, mask_final, view, count


def vertex_in_mask(screen, mask):
    """rint (half to even) of (col, row) inside the image and on a set mask pixel (texture_mesh_extract.py:89-95)."""
    H, W = mask.shape
    c, r = np.round(screen[:, 0]), np.round(screen[:, 1])
    inside = (c >= 0) & (c < W) & (r >= 0) & (r < H)
    out = np.zeros(screen.shape[0], bool)
    out[inside] = mask[r[inside].astype(np.int64), c[inside].astype(np.int64)] > 0
    return out
