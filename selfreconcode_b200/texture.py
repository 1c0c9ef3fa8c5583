"""Texture atlas of the reconstruction on the device: the reference's texture_mesh_prepare.py + texture_mesh_extract.py
(VideoAvatar's Isomapper aggregation) without pytorch3d, opendr or a second Python environment.

    V, F, vt, ft = load_obj_uv("template/uvmap.obj")
    baker = TextureBaker(F, vt, ft, resolution=1680, views=50, max_angle=68., min_views=5)
    for fid in texture_frame_ids(120, frame_num):
        baker.add_frame(deformed_verts, cameras, image_bgr, mask, fid)
    write_texture(out_dir, baker.finish())       # tex_mask.png, mask_final.png, tex_median.png, texture.png

or `bake_from_network(optNet, "template/uvmap.obj", out_dir)` from a trained network and its dataset.  The rule
(DESIGN.md section 3.3): every atlas texel covered by a UV face keeps the S best views of its point (weight = cosine
between the vertex normal and the view direction, interpolated over the face, above cos(max_angle)) among the frames
in which the face is visible and inside the mask; the texture is the per-channel median of those views' colours where
at least min_views were kept.  The per-texel work is csrc/texture_bake.cu; per-vertex and per-face flags are a few
torch ops over V and F."""
import math
import os
import os.path as osp

import numpy as np
import torch

from . import enable_dropin, ops

RATIO_ONE = {'sdfRatio': 1., 'deformerRatio': 1., 'renderRatio': 1.}


def load_obj_uv(path):
    """OBJ file -> (V [V,3] float32, F [F,3] int64, vt [T,2] float32, ft [F,3] int64), host tensors.  Reads `v`, `vt`
    and `f a/b[/c]` (other statements are ignored); indices are 1-based, or negative and counted from the end of the
    file's vertex / UV list, as pytorch3d's load_obj counts them; a polygon becomes the fan (0, i, i+1) as in
    pytorch3d's load_obj.  Raises ValueError on a face without UV indices or an index out of range."""
    verts, uvs, fv, ft = [], [], [], []
    with open(path, "r") as fh:
        for ln, line in enumerate(fh, 1):
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "vt":
                uvs.append([float(x) for x in tok[1:3]])
            elif tok[0] == "f":
                corners = []
                for c in tok[1:]:
                    parts = c.split("/")
                    if len(parts) < 2 or parts[1] == "":
                        raise ValueError("%s:%d: face without texture coordinates (%r)" % (path, ln, c))
                    corners.append((int(parts[0]), int(parts[1])))
                if len(corners) < 3:
                    raise ValueError("%s:%d: face with fewer than 3 vertices" % (path, ln))
                for i in range(len(corners) - 2):
                    tri = (corners[0], corners[i + 1], corners[i + 2])
                    fv.append([c[0] for c in tri])
                    ft.append([c[1] for c in tri])
    V = torch.tensor(verts, dtype=torch.float32).reshape(-1, 3)
    vt = torch.tensor(uvs, dtype=torch.float32).reshape(-1, 2)

    def index(a, n, what):
        t = torch.tensor(a, dtype=torch.int64).reshape(-1, 3)
        t = torch.where(t > 0, t - 1, t + n)         # 1-based; negative counts from the end
        if t.numel() and (bool((t < 0).any()) or bool((t >= n).any())):
            raise ValueError("%s: %s index out of range" % (path, what))
        return t
    return V, index(fv, V.shape[0], "vertex"), vt, index(ft, vt.shape[0], "texture coordinate")


def texture_frame_ids(num, frame_num):
    """The frames texturing uses: ceil(arange(num) * frame_num / num) (texture_mesh_prepare.py:81).  num must lie
    in [1, frame_num] (beyond it the formula indexes past the last frame)."""
    num, frame_num = int(num), int(frame_num)
    if num < 1 or num > frame_num:
        raise ValueError("texture_frame_ids: num must lie in [1, frame_num = %d], got %d" % (frame_num, num))
    return np.ceil(np.arange(num) * frame_num * 1. / num).astype(np.int64)


def _as_device(x, device, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else torch.as_tensor(x)
    return t.to(device=device, dtype=dtype if dtype is not None else t.dtype).contiguous()


def uv_raster(vt, ft, Ht, Wt):
    """UV faces on an Ht x Wt atlas: texel (i, j) is the pixel centre (col j, row i) of the screen vertices
    (u Wt - 0.5, (1-v) Ht - 0.5, 1).  vt [T,2] float32, ft [F,3] int64 device tensors -> (face [Ht,Wt] int64, -1 =
    uncovered; barycentrics [Ht,Wt,3])."""
    uv = torch.stack([vt[:, 0] * Wt - 0.5, (1. - vt[:, 1]) * Ht - 0.5, torch.ones_like(vt[:, 0])], dim=-1)
    p2f, bary, _ = ops.raster_mesh(uv[None], ft, Ht, Wt)
    return p2f.view(Ht, Wt), bary.view(Ht, Wt, 3)


class TextureBaker:
    """Streams frames into an R x R atlas with `views` slots per covered texel.  Device memory: 20 B per slot and
    covered texel (at most views * R^2 * 20 B: 2.8 GB at R = 1680 and 50 slots) plus 36 B per covered texel."""

    def __init__(self, faces, vt, ft, resolution=1680, views=50, max_angle=68., min_views=5, device="cuda"):
        R, S = int(resolution), int(views)
        if R <= 0:
            raise ValueError("TextureBaker: resolution must be positive, got %d" % R)
        if S <= 0 or S > ops.TEXTURE_MAX_SLOTS:
            raise ValueError("TextureBaker: views must lie in [1, %d], got %d" % (ops.TEXTURE_MAX_SLOTS, S))
        if not (0. < float(max_angle) < 90.):
            raise ValueError("TextureBaker: max_angle must lie in (0, 90) degrees, got %r" % (max_angle,))
        if not (1 <= int(min_views) <= S):
            raise ValueError("TextureBaker: min_views must lie in [1, views = %d], got %r" % (S, min_views))
        self.device = torch.device(device)
        self.R, self.S, self.min_views = R, S, int(min_views)
        self.c0 = float(np.float32(math.cos(math.radians(float(max_angle)))))
        self.faces = _as_device(faces, self.device, torch.int64).reshape(-1, 3)
        vt = _as_device(vt, self.device, torch.float32).reshape(-1, 2)
        ft = _as_device(ft, self.device, torch.int64).reshape(-1, 3)
        if ft.shape != self.faces.shape:
            raise ValueError("TextureBaker: ft must have one row per face (%d), got %d" % (self.faces.shape[0], ft.shape[0]))
        p2f, bary = uv_raster(vt, ft, R, R)
        p2f, bary = p2f.view(R * R), bary.view(R * R, 3)
        self.tex_mask = (p2f >= 0).view(R, R)
        self.texel_index = torch.nonzero(p2f >= 0).view(-1)
        self.texel_face = p2f[self.texel_index].to(torch.int32).contiguous()
        self.texel_bary = bary[self.texel_index].contiguous()
        T = self.texel_index.numel()
        if T == 0:
            raise ValueError("TextureBaker: no atlas texel is covered by a UV face")
        self.slots = dict(rgb=torch.zeros((S, 3, T), dtype=torch.float32, device=self.device),
                          alpha=torch.full((S, T), self.c0, dtype=torch.float32, device=self.device),
                          view=torch.full((S, T), -1, dtype=torch.int32, device=self.device),
                          min_alpha=torch.full((T,), self.c0, dtype=torch.float32, device=self.device),
                          min_slot=torch.zeros((T,), dtype=torch.int32, device=self.device))
        self._csr = None

    def _vertex_csr(self, V):
        if self._csr is None or self._csr[0] != V:
            enable_dropin()
            from model.raster import vertex_face_csr
            self._csr = (V, vertex_face_csr(self.faces, V))
        return self._csr[1]

    def frame_inputs(self, def_verts, cameras, mask):
        """One frame's per-vertex and per-face inputs of the accumulation: (screen vertices [V,3] = (col, row, Z),
        vertex weights a_v = max(0, -n_v . d_v) [V], usable-face flags [F] uint8).  A face is usable when its three
        vertices round (half to even) into the mask and it owns a pixel of the frame's mesh raster."""
        enable_dropin()
        from model.raster import screen_vertices
        with torch.no_grad():
            D = def_verts.detach().to(self.device, torch.float32).reshape(1, -1, 3).contiguous()
            V = D.shape[1]
            m = _as_device(mask, self.device).bool()
            H, W = m.shape
            s = screen_vertices(D, cameras).contiguous()
            col, row = torch.round(s[0, :, 0]), torch.round(s[0, :, 1])
            inview = (col >= 0) & (col < W) & (row >= 0) & (row < H)
            ci = torch.where(inview, col, torch.zeros_like(col)).long()
            ri = torch.where(inview, row, torch.zeros_like(row)).long()
            in_mask = inview & m[ri, ci]
            p2f, _, _ = ops.raster_mesh(s, self.faces, H, W)
            F = self.faces.shape[0]
            ids = p2f.view(-1)
            owned = torch.zeros(F + 1, dtype=torch.bool, device=self.device)
            owned.index_fill_(0, torch.where(ids >= 0, ids, torch.full_like(ids, F)), True)
            usable = (in_mask[self.faces].all(1) & owned[:F]).to(torch.uint8)
            normals = ops.mesh_vertex_normals(D, self.faces, self._vertex_csr(V))[0]
            d = torch.nn.functional.normalize(D[0] - cameras.cam_pos(0).to(D).view(1, 3), dim=1)
            weight = (-(normals * d).sum(1)).clamp(min=0.).contiguous()
        return s[0], weight, usable

    def accumulate(self, screen, weight, usable, image, frame_id):
        """The per-texel step of add_frame on given frame inputs (see frame_inputs)."""
        img = _as_device(image, self.device, torch.uint8)
        ops.texture_accumulate(self.texel_face, self.texel_bary, screen.contiguous(), self.faces, weight.contiguous(),
                               usable.contiguous(), img, int(frame_id), self.slots)

    def add_frame(self, def_verts, cameras, image, mask, frame_id):
        """def_verts [V,3] (or [1,V,3]) deformed template of the frame, cameras = its RectifiedPerspectiveCameras
        (camera 0 is used), image [H,W,3] uint8 (BGR as cv2 reads it), mask [H,W] (nonzero = foreground), frame_id >= 0
        recorded in view_id.  Frames are applied in call order."""
        if int(frame_id) < 0:
            raise ValueError("TextureBaker.add_frame: frame_id must be >= 0")
        img = _as_device(image, self.device, torch.uint8)
        if img.dim() != 3 or img.shape[2] != 3 or tuple(img.shape[:2]) != tuple(mask.shape):
            raise ValueError("TextureBaker.add_frame: image must be [H,W,3] and mask [H,W] of the same size")
        screen, weight, usable = self.frame_inputs(def_verts, cameras, mask)
        self.accumulate(screen, weight, usable, img, frame_id)

    def finish(self):
        """-> dict of device tensors: tex_median [R,R,3] float32 in [0,1] (image channel order), mask_final [R,R] bool,
        tex_mask [R,R] bool, view_id [R,R] int32 (-1 where not mask_final), count [R,R] int32."""
        R = self.R
        med, mask, view, count = ops.texture_finish(self.texel_index, self.slots, self.c0, self.min_views, R * R)
        return dict(tex_median=med.view(R, R, 3), mask_final=mask.view(R, R).bool(), tex_mask=self.tex_mask,
                    view_id=view.view(R, R), count=count.view(R, R))


def write_texture(out_dir, result):
    """Writes tex_mask.png, mask_final.png, tex_median.png and texture.png (the median with the unseen texels near
    the atlas charts Telea-inpainted, texture_mesh_extract.py:135-153) into out_dir."""
    import cv2
    os.makedirs(out_dir, exist_ok=True)
    tex_mask = result["tex_mask"].cpu().numpy().astype(np.float32)
    mask_final = result["mask_final"].cpu().numpy().astype(np.float32)
    med = np.uint8(result["tex_median"].cpu().numpy().astype(np.float64) * 255)
    cv2.imwrite(osp.join(out_dir, "tex_mask.png"), np.uint8(tex_mask * 255))
    cv2.imwrite(osp.join(out_dir, "mask_final.png"), np.uint8(mask_final * 255))
    cv2.imwrite(osp.join(out_dir, "tex_median.png"), med)
    k = int(tex_mask.shape[0] * 0.1)
    inpaint_area = cv2.dilate(tex_mask, np.ones((k, k), np.uint8)) - mask_final
    cv2.imwrite(osp.join(out_dir, "texture.png"), cv2.inpaint(med, np.uint8(inpaint_area * 255), 3, cv2.INPAINT_TELEA))


def _read_frame(names, fid, what):
    import cv2
    path = names[fid]
    if not osp.isfile(path) or int(osp.basename(path).split(".")[0]) != fid:
        raise ValueError("bake_from_network: %s file of frame %d is %r" % (what, fid, path))
    return cv2.imread(path)


def bake_from_network(optNet, uv_obj_path, out_dir, num=120, resolution=1680, views=50, max_angle=68., min_views=5,
                      batch=8, device=None):
    """texture_mesh_prepare.py + texture_mesh_extract.py end to end: deforms the UV template (uvmap.obj) with
    optNet.deformer at ratio 1 for `num` frames of optNet.dataset, bakes them in order and writes the four images into
    out_dir.  Returns finish()'s dict."""
    enable_dropin()
    from model.CameraMine import RectifiedPerspectiveCameras
    dataset = optNet.dataset
    if device is None:
        device = next(optNet.deformer.parameters()).device
    V, F, vt, ft = load_obj_uv(uv_obj_path)
    fids = texture_frame_ids(num, dataset.frame_num)
    baker = TextureBaker(F, vt, ft, resolution, views, max_angle, min_views, device)
    f, pp, R, T, _, _ = dataset.get_camera_parameters(1, device)
    cams = RectifiedPerspectiveCameras(f.detach(), pp.detach(), R.detach(), T.detach())
    TmpVs = V.to(device)
    for b in range(0, len(fids), int(batch)):
        ids = torch.as_tensor(fids[b:b + int(batch)], dtype=torch.int64)
        with torch.no_grad():
            poses, trans, d_cond = dataset.get_grad_parameters(ids, device)[:3]
            defVs = optNet.deformer(TmpVs[None].expand(ids.numel(), -1, 3), [d_cond, [poses, trans]], ratio=RATIO_ONE)
        for k, fid in enumerate(ids.tolist()):
            image = _read_frame(dataset.img_ns, fid, "image")
            mask = _read_frame(dataset.mask_ns, fid, "mask")
            mask = mask.any(-1) if mask.ndim > 2 else mask > 0
            baker.add_frame(defVs[k], cams, image, mask, fid)
    result = baker.finish()
    write_texture(out_dir, result)
    return result
