"""The textured avatar on the device: the UV template (uvmap.obj) with its baked atlas (texture.png), reposed by the
trained deformer and rendered under the sequence's camera, plus an export that animates it without this package.

    avatar = TexturedAvatar("template/uvmap.obj", "template/texture.png")
    render_sequence(optNet, avatar, "textured")                        # every frame over its image, errors.txt
    d = np.load("other/smpl_rec.npz")
    render_motion(optNet, avatar, "motion", d["poses"], d["trans"])    # another sequence's poses
    export_avatar(optNet, avatar, "avatar.npz")                        # template, UVs, skin weights, skeleton

optNet is a trained OptimNetwork loaded as infer.py loads it, with its dataset attached (as texture.bake_from_network
reads it).  Posing goes through optNet.deformer at ratio 1 (translator, then the skinner); rendering is the built-in
rasteriser plus csrc/avatar_texture.cu: an unlit, trilinear-filtered lookup in a coverage-weighted mip pyramid of the
atlas (DESIGN.md section 3.3).  Frames go through the device in batches; image and video encoding run on a host thread
pool."""
import os
import os.path as osp
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import enable_dropin, ops
from .texture import RATIO_ONE, load_obj_uv, uv_raster


def _read_atlas(texture):
    if isinstance(texture, (str, os.PathLike)):
        import cv2
        img = cv2.imread(str(texture), cv2.IMREAD_UNCHANGED)
        if img is None:
            raise ValueError("TexturedAvatar: cannot read the atlas %r" % (texture,))
    else:
        img = np.asarray(texture)
    if img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.uint8 or img.shape[0] == 0 or img.shape[1] == 0:
        raise ValueError("TexturedAvatar: the atlas must be [Ht,Wt,3] uint8, got %s %s" % (img.shape, img.dtype))
    return np.ascontiguousarray(img)


class TexturedAvatar:
    """V [V,3], faces / ft [F,3], vt [T,2] of the UV template and the atlas [Ht,Wt,3] uint8 (BGR as cv2 reads it) on
    the device, with its mip pyramid (mips, levels of ops.texture_mips) built once.  The pyramid's level-0 coverage is
    the UV raster of ft at the atlas size: the baker's tex_mask.  texture_png may also be an [Ht,Wt,3] uint8 array."""

    def __init__(self, uvmap_obj, texture_png, device="cuda"):
        atlas = _read_atlas(texture_png)
        V, F, vt, ft = load_obj_uv(uvmap_obj)
        self.device = torch.device(device)
        self.texture_name = osp.basename(str(texture_png)) if isinstance(texture_png, (str, os.PathLike)) \
            else "texture.png"
        self.V, self.faces = V.to(self.device), F.to(self.device)
        self.vt, self.ft = vt.to(self.device), ft.to(self.device)
        self.atlas = torch.from_numpy(atlas).to(self.device)
        Ht, Wt = atlas.shape[:2]
        self.coverage = uv_raster(self.vt, self.ft, Ht, Wt)[0] >= 0
        self.mips, self.levels = ops.texture_mips(self.atlas, self.coverage)


def _as_tensor(x, what):
    try:
        return x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))
    except (TypeError, ValueError):
        raise ValueError("%s must be an array" % what)


def motion_args(poses, trans, yaw_deg=None):
    """poses [T,24,3] or [T,72] (the smpl_rec.npz layout), trans [T,3], yaw_deg [T] or None -> (poses [T,24,3],
    trans [T,3], yaw_deg) as float32 tensors on their own device; ValueError on any other shape."""
    p = _as_tensor(poses, "poses")
    if not ((p.dim() == 3 and tuple(p.shape[1:]) == (24, 3)) or (p.dim() == 2 and p.shape[1] == 72)) or p.shape[0] == 0:
        raise ValueError("poses must be [T,24,3] or [T,72], got %s" % (tuple(p.shape),))
    T = p.shape[0]
    t = _as_tensor(trans, "trans")
    if tuple(t.shape) != (T, 3):
        raise ValueError("trans must be [T,3] = [%d,3] like the poses, got %s" % (T, tuple(t.shape)))
    y = None
    if yaw_deg is not None:
        y = _as_tensor(yaw_deg, "yaw_deg")
        if y.numel() != T:
            raise ValueError("yaw_deg must hold one angle per pose (%d), got %d" % (T, y.numel()))
        y = y.reshape(T).to(torch.float64)
    return p.reshape(T, 24, 3).to(torch.float32), t.to(torch.float32), y


def _check_cond_frame(optNet, cond_frame):
    n = int(optNet.dataset.frame_num)
    if not (0 <= int(cond_frame) < n):
        raise ValueError("cond_frame must lie in [0, %d), got %r" % (n, cond_frame))
    return int(cond_frame)


def _device(optNet):
    return next(optNet.deformer.parameters()).device


def _cameras(optNet, n, device):
    enable_dropin()
    from model.CameraMine import RectifiedPerspectiveCameras
    f, pp, R, T, _, _ = optNet.dataset.get_camera_parameters(n, device)
    return RectifiedPerspectiveCameras(f.detach(), pp.detach(), R.detach(), T.detach())


def pose_vertices(optNet, V, poses, trans, d_cond, yaw_deg=None):
    """The template V [V,3] posed by optNet.deformer at ratio 1 for T poses -> [T,V,3].  poses [T,24,3] or [T,72],
    trans [T,3], d_cond [T,C] translator codes (or one code [C] / [1,C] for every pose).  yaw_deg [T] (optional) then
    turns each posed mesh about the camera's vertical image axis through the frame's posed root joint (Js[0] + trans:
    the skeleton's root transform keeps the root joint in place), a turntable for one pose repeated with
    yaw = linspace(0, 360, K); a zero angle leaves the vertices bit-identical."""
    poses, trans, yaw = motion_args(poses, trans, yaw_deg)
    dev = V.device
    T = poses.shape[0]
    poses, trans = poses.to(dev), trans.to(dev)
    d = _as_tensor(d_cond, "d_cond").to(dev)
    if d.dim() == 1:
        d = d.view(1, -1)
    if d.shape[0] == 1 and T > 1:
        d = d.expand(T, -1).contiguous()
    if d.dim() != 2 or d.shape[0] != T:
        raise ValueError("d_cond must be [T,C] or one code, got %s for %d poses" % (tuple(d.shape), T))
    with torch.no_grad():
        out = optNet.deformer(V[None].expand(T, -1, 3), [d, [poses, trans]], ratio=RATIO_ONE)
        if yaw is None:
            return out
        R = optNet.dataset.get_camera_parameters(1, dev)[2]
        axis = R.detach().reshape(3, 3)[:, 1].double()          # camera y (image rows) in world: p_cam = p R + T
        axis = axis / axis.norm()
        centre = (optNet.deformer.defs[-1].Js[0].double() + trans.double()).view(T, 1, 3)
        th = torch.deg2rad(yaw.to(dev))
        p = out.double()
        a = axis.view(1, 1, 3).expand_as(p)
        axd = torch.cross(a, p - centre, dim=-1)
        # Rodrigues about the axis through the root, as p + sin(t) a x d + (1 - cos(t)) a x (a x d): exactly p at t = 0
        p = p + torch.sin(th).view(T, 1, 1) * axd + (1. - torch.cos(th)).view(T, 1, 1) * torch.cross(a, axd, dim=-1)
        return p.float()


def _render(avatar, verts, cams, H, W, background):
    """Posed vertices [B,V,3] -> (images [B,H,W,3] uint8 in the atlas' channel order, coverage [B,H,W] bool)."""
    from model.raster import screen_vertices
    s = screen_vertices(verts, cams).contiguous()
    p2f, bary, _ = ops.raster_mesh(s, avatar.faces, H, W)
    out = ops.shade_textured(p2f[..., 0], bary[..., 0, :], s, avatar.faces, avatar.ft, avatar.vt, avatar.mips,
                             avatar.levels, background)
    return torch.round(out[..., :3].clamp(0., 1.) * 255.).to(torch.uint8), p2f[..., 0] >= 0


def _read_frame(path, fid, what):
    import cv2
    if not osp.isfile(path) or int(osp.basename(path).split(".")[0]) != fid:
        raise ValueError("render_sequence: %s file of frame %d is %r" % (what, fid, path))
    return cv2.imread(path)


def _read_pair(ds, fid):
    img = _read_frame(ds.img_ns[fid], fid, "image")
    m = _read_frame(ds.mask_ns[fid], fid, "mask")
    return img, (m.any(-1) if m.ndim > 2 else m > 0)


def frame_errors(render, frame, mask):
    """Photometric error of rendered frames over the pixels both covered (mask [B,H,W] bool: coverage & the frame's
    mask): (mean |render - frame| in 0..255 units [B], PSNR in dB [B]) as float64; -1 / -1 for a frame without such
    pixels.  render / frame [B,H,W,3] uint8 device tensors."""
    d = (render.to(torch.int32) - frame.to(torch.int32)).to(torch.float64) * mask[..., None]
    cnt = mask.sum((1, 2)).to(torch.float64) * 3.
    mad = d.abs().sum((1, 2, 3)) / cnt
    psnr = 10. * torch.log10(255. ** 2 / ((d * d).sum((1, 2, 3)) / cnt))
    none = cnt == 0
    return torch.where(none, -1., mad), torch.where(none, -1., psnr)


def _write_errors(path, fids, mad, psnr):
    with open(path, "w") as fh:
        fh.write("         mad     psnr\n")
        for i, m, p in zip(fids, mad, psnr):
            if m >= 0.:
                fh.write("%4d: %.4f %.4f\n" % (i, m, p))
        ok = mad >= 0.
        for name, e, worst in (("mad", mad[ok], -mad[ok]), ("psnr", psnr[ok], psnr[ok])):
            if e.size == 0:
                continue
            fh.write("%s mean: %.4f, max: %.4f, min: %.4f, worstinds:" % (name, e.mean(), e.max(), e.min()))
            fh.write("".join(" %d" % i for i in np.asarray(fids)[ok][np.argsort(worst, kind="stable")[:10]]) + "\n")


class _Writer:
    """PNG files on a thread pool, video frames in order on a thread of their own (cv2 mp4v, 30 fps)."""

    def __init__(self, out_dir, H, W):
        import cv2
        os.makedirs(out_dir, exist_ok=True)
        self.dir = out_dir
        self.pool = ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1))
        self.vpool = ThreadPoolExecutor(max_workers=1)
        self.video = cv2.VideoWriter(osp.join(out_dir, "video.mp4"), cv2.VideoWriter.fourcc(*"mp4v"), 30., (W, H))
        self.pending = []

    def put(self, name, img):
        import cv2
        self.pending.append(self.pool.submit(cv2.imwrite, osp.join(self.dir, "%d.png" % name), img))
        self.pending.append(self.vpool.submit(self.video.write, img))

    def close(self):
        try:
            for f in self.pending:
                f.result()
        finally:
            self.vpool.shutdown()
            self.pool.shutdown()
            self.video.release()


def render_sequence(optNet, avatar, out_dir, frames=None, batch=8):
    """Renders the sequence's own frames (each with its pose, translation and translator code) textured over the
    frame image and writes out_dir/%d.png, video.mp4 and errors.txt: per frame the mean absolute difference (0..255)
    and the PSNR between render and image over the pixels covered by the render and inside the frame's mask, then
    mean / max / min lines.  Returns (frame ids, mad, psnr) as numpy arrays."""
    enable_dropin()
    ds = optNet.dataset
    n = int(ds.frame_num)
    fids = np.arange(n) if frames is None else np.asarray(frames, np.int64).reshape(-1)
    if fids.size == 0 or fids.min() < 0 or fids.max() >= n:
        raise ValueError("render_sequence: frames must lie in [0, %d)" % n)
    B = int(batch)
    if B <= 0:
        raise ValueError("render_sequence: batch must be positive")
    dev = _device(optNet)
    H, W = int(ds.H), int(ds.W)
    cams = _cameras(optNet, B, dev)
    out = _Writer(out_dir, H, W)
    mads, psnrs = [], []
    reader = ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1))
    try:
        ahead = [reader.submit(_read_pair, ds, int(f)) for f in fids[:2 * B]]      # decoded ahead of the device
        for b in range(0, fids.size, B):
            ids = fids[b:b + B]
            pairs = [f.result() for f in ahead[:ids.size]]
            ahead = ahead[ids.size:] + [reader.submit(_read_pair, ds, int(f)) for f in fids[b + 2 * B:b + 2 * B + ids.size]]
            frame = torch.from_numpy(np.stack([p[0] for p in pairs])).to(dev)
            mask = torch.from_numpy(np.stack([p[1] for p in pairs])).to(dev)
            if tuple(frame.shape[1:3]) != (H, W):
                raise ValueError("render_sequence: frame images must be %d x %d" % (H, W))
            poses, trans, d_cond = ds.get_grad_parameters(torch.as_tensor(ids, dtype=torch.int64), dev)[:3]
            verts = pose_vertices(optNet, avatar.V, poses, trans, d_cond)
            img, cov = _render(avatar, verts, cams, H, W, frame)
            mad, psnr = frame_errors(img, frame, cov & mask)
            host = img.cpu().numpy()
            for k, fid in enumerate(ids.tolist()):
                out.put(fid, host[k])
            mads.append(mad.cpu().numpy())
            psnrs.append(psnr.cpu().numpy())
    finally:
        reader.shutdown()
        out.close()
    mad, psnr = np.concatenate(mads), np.concatenate(psnrs)
    _write_errors(osp.join(out_dir, "errors.txt"), fids, mad, psnr)
    return fids, mad, psnr


def render_motion(optNet, avatar, out_dir, poses, trans, cond_frame=0, yaw_deg=None, background=(1., 1., 1.),
                  batch=8):
    """Renders new poses (poses [T,24,3] or [T,72], trans [T,3], e.g. another sequence's smpl_rec.npz) under the
    sequence's camera and image size over a constant background (3 floats in [0,1], atlas channel order), and writes
    out_dir/%d.png (0..T-1) and video.mp4.  Every frame uses the translator code of cond_frame: the non-rigid offset
    is frozen at that frame's, so the clothing dynamics of new poses are not predicted.  yaw_deg [T] as in
    pose_vertices."""
    poses, trans, yaw = motion_args(poses, trans, yaw_deg)
    cond_frame = _check_cond_frame(optNet, cond_frame)
    B = int(batch)
    if B <= 0:
        raise ValueError("render_motion: batch must be positive")
    bg = [float(c) for c in background]
    if len(bg) != 3:
        raise ValueError("render_motion: background must be 3 floats")
    enable_dropin()
    ds = optNet.dataset
    dev = _device(optNet)
    H, W = int(ds.H), int(ds.W)
    cams = _cameras(optNet, B, dev)
    d_cond = ds.get_grad_parameters(torch.tensor([cond_frame], dtype=torch.int64), dev)[2]
    out = _Writer(out_dir, H, W)
    try:
        for b in range(0, poses.shape[0], B):
            sl = slice(b, b + B)
            verts = pose_vertices(optNet, avatar.V, poses[sl], trans[sl], d_cond, None if yaw is None else yaw[sl])
            host = _render(avatar, verts, cams, H, W, bg)[0].cpu().numpy()
            for k in range(host.shape[0]):
                out.put(b + k, host[k])
    finally:
        out.close()


def rest_inverse(skinner):
    """[24,4,4] float64: the map from the canonical template into each bone's rest frame, so that linear blend
    skinning is A_j = G_j @ rest_inverse_j with G_j the posed chain: the skinner's init_pose, or [I, -Js_j] without
    one."""
    if skinner.init_pose is not None:
        return skinner.init_pose.detach().double().cpu().view(24, 4, 4).numpy()
    inv = np.tile(np.eye(4), (24, 1, 1))
    inv[:, :3, 3] = -skinner.Js.detach().double().cpu().numpy().reshape(24, 3)
    return inv


def export_avatar(optNet, avatar, path, cond_frame=0):
    """Writes an .npz that animates the textured template without this package: verts [V,3] (the UV template plus the
    translator offset of cond_frame), faces [F,3], vt [T,2], ft [F,3], skin_weights [V,24] (the skinner's volume
    sampled at verts by the device trilinear sampler), Js [24,3], parents [24], init_pose [24,4,4] (rest_inverse) and
    texture (the atlas' file name).  Linear blend skinning with them,
        G_j = G_parent(j) [R(pose_j), Js_j - Js_parent(j)] (G_0 = [R(pose_0), Js_0]),  A_j = G_j init_pose_j,
        v' = (sum_j w_vj A_j) [v, 1] + trans,
    reproduces optNet.deformer for that frame's translator code."""
    cond_frame = _check_cond_frame(optNet, cond_frame)
    ds = optNet.dataset
    dev = avatar.V.device
    tr, sk = optNet.deformer.defs[0], optNet.deformer.defs[-1]
    d_cond = ds.get_grad_parameters(torch.tensor([cond_frame], dtype=torch.int64), dev)[2]
    with torch.no_grad():
        verts = tr(avatar.V[None].contiguous(), d_cond, ratio=RATIO_ONE).reshape(-1, 3).float().contiguous()
        nps = 2. * (verts - sk.b_min.view(1, 3)) / (sk.b_max - sk.b_min).view(1, 3) - 1.
        ws = ops.grid_sample3d_forward(sk.ws.contiguous(), nps.view(1, 1, 1, -1, 3).contiguous())
        ws = ws.view(ws.shape[1], -1).t()
    np.savez(path, verts=verts.cpu().numpy(), faces=avatar.faces.cpu().numpy(), vt=avatar.vt.cpu().numpy(),
             ft=avatar.ft.cpu().numpy(), skin_weights=ws.cpu().numpy(),
             Js=sk.Js.detach().float().cpu().numpy().reshape(24, 3),
             parents=np.asarray([int(p) for p in sk.parents], np.int64),
             init_pose=rest_inverse(sk).astype(np.float32), texture=np.array(avatar.texture_name))
