"""Seeded synthetic workloads for the hot path (SURVEY.md section 8d).

No assets are needed: the networks use the reference's own initialisers under a fixed seed
(geometric init makes the SDF a radius-0.6 sphere, model/network.py:49-63) plus a small
perturbation; the skin-weight volume is a softmax of Gaussian blobs around a synthetic
24-joint tree; the camera follows the PeopleSnapshot convention.  Everything is built on the
CPU generator (bit-reproducible across machines) and then moved to the requested device.
"""
import math

import numpy as np
import torch

from . import enable_dropin

enable_dropin()
from model.network import ImplicitNetwork  # noqa: E402
from model.Deformer import MLPTranslator, LBSkinner, CompositeDeformer  # noqa: E402
from model.RenderNet import RenderingNetwork_view_norm  # noqa: E402

# SMPL kinematic tree (parents[0] is unused)
SMPL_PARENTS = np.array([0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19,
                         20, 21], dtype=np.int64)
# approximate SMPL rest joints (metres), only used to place the synthetic blobs
SYNTH_JOINTS = np.array([
    [0.00, -0.22, 0.00], [0.07, -0.31, 0.00], [-0.07, -0.31, 0.00], [0.00, -0.10, -0.02],
    [0.10, -0.70, 0.00], [-0.10, -0.70, 0.00], [0.00, 0.04, 0.00], [0.09, -1.10, -0.03],
    [-0.09, -1.10, -0.03], [0.00, 0.10, 0.00], [0.11, -1.16, 0.09], [-0.11, -1.16, 0.09],
    [0.00, 0.31, -0.03], [0.08, 0.22, -0.02], [-0.08, 0.22, -0.02], [0.00, 0.40, 0.02],
    [0.19, 0.25, -0.03], [-0.19, 0.25, -0.03], [0.45, 0.24, -0.04], [-0.45, 0.24, -0.04],
    [0.70, 0.24, -0.04], [-0.70, 0.24, -0.04], [0.79, 0.23, -0.05], [-0.79, 0.23, -0.05]],
    dtype=np.float32)
B_MIN = (-0.9, -1.3, -0.5)
B_MAX = (0.9, 0.9, 0.5)


def _perturb(module, scale, gen):
    if scale <= 0:
        return
    with torch.no_grad():
        for p in module.parameters():
            p.add_(scale * torch.randn(p.shape, generator=gen))


def make_sdf(seed=0, hidden=512, n_hidden=8, multires=6, feat=256, skip_in=(4,), perturb=3e-3,
             bias=0.78):
    """8x512 SDF, skip at 4, 256-d feature.  bias 0.78 + 3e-3 weight noise give a lumpy sphere of
    mean radius ~0.6 (radius std ~0.07).  (SURVEY.md 8d suggested bias 0.6 / noise 1e-2; with
    PE + softplus(100) that zero set sits at r~0.34 and 1e-2 noise on every weight removes it
    -- the reference would assert "tmp sdf vanished", network.py:466-468.)"""
    torch.manual_seed(seed)
    net = ImplicitNetwork(feat, 3, 1, [hidden] * n_hidden, geometric_init=True, bias=bias,
                          skip_in=list(skip_in), weight_norm=True, multires=multires)
    _perturb(net, perturb, torch.Generator().manual_seed(seed + 1000))
    return net


def make_translator(seed=1, condlen=128, multires=6, perturb=1e-2):
    torch.manual_seed(seed)
    net = MLPTranslator(condlen, multires)
    _perturb(net, perturb, torch.Generator().manual_seed(seed + 1000))
    return net


def make_render(seed=2, condlen=256, multires_v=4):
    torch.manual_seed(seed)
    return RenderingNetwork_view_norm(condlen, d_in=9, d_out=3, dims=[512] * 4, mode='idr',
                                      weight_norm=True, multires_v=multires_v, multires_n=0)


def smpl_apose(kind=1):
    pose = np.zeros((24, 3), dtype=np.float32)
    leg, arm = {0: (10., 45.), 1: (7., 55.)}[kind]
    pose[1, 2] = leg / 180. * np.pi
    pose[2, 2] = -leg / 180. * np.pi
    pose[16, 2] = -arm / 180. * np.pi
    pose[17, 2] = arm / 180. * np.pi
    return pose


def make_skinner(seed=3, resolution=(129, 225, 65), sigma=0.18):
    """LBSkinner over a synthetic weight volume [1,24,D,H,W] (W,H,D = resolution)."""
    W, H, D = resolution
    bmin = torch.tensor(B_MIN)
    bmax = torch.tensor(B_MAX)
    Js = torch.from_numpy(SYNTH_JOINTS.copy())
    # voxel centres, align_corners=False convention (model/Deformer.py:256-261)
    xs = (torch.arange(W).float() + 0.5) / W * (bmax[0] - bmin[0]) + bmin[0]
    ys = (torch.arange(H).float() + 0.5) / H * (bmax[1] - bmin[1]) + bmin[1]
    zs = (torch.arange(D).float() + 0.5) / D * (bmax[2] - bmin[2]) + bmin[2]
    logits = torch.empty(24, D, H, W)
    for j in range(24):
        d2 = ((zs - Js[j, 2]) ** 2).view(D, 1, 1) + ((ys - Js[j, 1]) ** 2).view(1, H, 1) + \
             ((xs - Js[j, 0]) ** 2).view(1, 1, W)
        logits[j] = -d2 / (2 * sigma * sigma)
    ws = torch.softmax(logits, dim=0).unsqueeze(0).contiguous()
    return LBSkinner(ws, list(B_MIN), list(B_MAX), Js, SMPL_PARENTS, init_pose=smpl_apose(1),
                     align_corners=False)


def make_frame_params(seed, n_frames, condlen=128, pose_sigma=0.2, trans_sigma=0.05):
    g = torch.Generator().manual_seed(seed)
    poses = pose_sigma * torch.randn(n_frames, 24, 3, generator=g)
    trans = trans_sigma * torch.randn(n_frames, 3, generator=g)
    dcond = 0.1 * torch.randn(n_frames, condlen, generator=g)
    return poses, trans, dcond


def camera(H, W):
    """PeopleSnapshot-style pinhole: fx=fy=W, principal point at the centre,
    R = quat2mat((0,0,0,1)) = diag(-1,-1,1), T = (0,0,2.5)  (SURVEY.md 8d)."""
    focal = torch.tensor([float(W), float(W)])
    pp = torch.tensor([W / 2.0, H / 2.0])
    R = torch.diag(torch.tensor([-1.0, -1.0, 1.0]))
    T = torch.tensor([0.0, 0.0, 2.5])
    cam_pos = -R.matmul(T.view(3, 1)).view(3)  # model/CameraMine.py:169-170
    return dict(focal=focal, pp=pp, R=R, T=T, cam_pos=cam_pos, H=H, W=W)


def view_rays(cam, cols, rows):
    """model/CameraMine.py:129-136 on pixel (col,row,1)."""
    fx, fy = cam["focal"][0], cam["focal"][1]
    cx, cy = cam["pp"][0], cam["pp"][1]
    r = torch.stack([-cols / fx + cx / fx, -rows / fy + cy / fy, torch.ones_like(cols)], dim=1)
    r = r / r.norm(dim=1, keepdim=True)
    return r.matmul(cam["R"].t())


def sphere_pixels(cam, radius=0.6):
    """All pixels whose ray hits the radius-`radius` sphere at the origin, and the hit points."""
    H, W = cam["H"], cam["W"]
    rows, cols = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    rows, cols = rows.reshape(-1), cols.reshape(-1)
    v = view_rays(cam, cols, rows)
    c = cam["cam_pos"].view(1, 3)
    b = (v * c).sum(1)
    disc = b * b - ((c * c).sum() - radius * radius)
    hit = disc > 0
    t = -b[hit] - torch.sqrt(disc[hit])
    pts = c + t.view(-1, 1) * v[hit]
    return rows[hit].long(), cols[hit].long(), pts


def project_to_surface(sdf_fn, dirs, lo=0.05, hi=1.5, iters=40, chunk=65536):
    """Bisection along each unit direction onto the SDF's zero level set (setup only)."""
    out = []
    for d in torch.split(dirs, chunk):
        a = torch.full((d.shape[0],), lo)
        b = torch.full((d.shape[0],), hi)
        for _ in range(iters):
            mid = (a + b) / 2
            f = sdf_fn(mid.view(-1, 1) * d).detach().cpu().view(-1)
            a, b = torch.where(f < 0, mid, a), torch.where(f < 0, b, mid)
        out.append(((a + b) / 2).view(-1, 1) * d)
    return torch.cat(out, 0)


def make_rays(cam, n_frames, sdf_fn, deform_fn, seed=7, jitter=5e-3, radius=0.6, max_rays=None):
    """Per-frame ray set: one ray per silhouette pixel of the radius-`radius` sphere.  The pixel's
    analytic hit direction is projected onto the SDF's actual zero set (p*), and the ray is
    re-aimed through D(p*) so that the constraint {f=0, (D(p)-c) x v=0} has its solution at p*
    (in the real pipeline the start point comes from rasterising the *deformed* mesh,
    utils/FindSurfacePs.py:5-29); starts are p* + N(0, jitter).
    sdf_fn(points [P,3]) -> [P];  deform_fn(points [P,3], batch_inds [P]) -> [P,3]; both may run
    on any device (CPU tensors in, any device out)."""
    rows, cols, pts = sphere_pixels(cam, radius)
    n = pts.shape[0]
    g = torch.Generator().manual_seed(seed)
    if max_rays is not None and n > max_rays:
        sel = torch.randperm(n, generator=g)[:max_rays].sort()[0]
        rows, cols, pts = rows[sel], cols[sel], pts[sel]
        n = max_rays
    pts = project_to_surface(sdf_fn, pts / pts.norm(dim=1, keepdim=True))
    batch = torch.arange(n_frames).view(-1, 1).expand(n_frames, n).reshape(-1).clone()
    pstar = pts.repeat(n_frames, 1)
    rows_all = rows.repeat(n_frames)
    cols_all = cols.repeat(n_frames)
    d = deform_fn(pstar, batch).detach().cpu()
    v = d - cam["cam_pos"].view(1, 3)
    v = v / v.norm(dim=1, keepdim=True)
    start = pstar + jitter * torch.randn(pstar.shape, generator=g)
    return dict(batch_inds=batch, rows=rows_all, cols=cols_all, rays=v, init_pts=start,
                pstar=pstar)


def ang_threshold(cam, pixoffset=0.5):
    """model/CameraMine.py:145-167 angThreshold (degrees)."""
    H, W = cam["H"], cam["W"]
    cx, cy = cam["pp"][0].item(), cam["pp"][1].item()
    fx, fy = cam["focal"][0].item(), cam["focal"][1].item()

    def ang(a, b):
        r1 = torch.tensor(a)
        r2 = torch.tensor(b)
        return torch.arcsin(torch.linalg.cross(r1, r2).norm() / (r1.norm() * r2.norm())) / np.pi * 180.

    th = ang([(W - cx) / fx, 0., 1.], [(W + pixoffset - cx) / fx, 0., 1.])
    th = torch.min(th, ang([-cx / fx, 0., 1.], [(pixoffset - cx) / fx, 0., 1.]))
    th = torch.min(th, ang([0., (H - cy) / fy, 1.], [0., (H + pixoffset - cy) / fy, 1.]))
    th = torch.min(th, ang([0., -cy / fy, 1.], [0., (pixoffset - cy) / fy, 1.]))
    return th.item()


# MC ladders (train.py:55-61 `resolutions_higher`, truncated as SURVEY.md 8d says)
MC_LADDER_257 = [(33, 33, 33), (65, 65, 65), (129, 129, 129), (257, 257, 257)]
MC_LADDER_513 = MC_LADDER_257 + [(513, 513, 513)]
MC_LADDER_65 = [(9, 9, 9), (17, 17, 17), (33, 33, 33), (65, 65, 65)]
MC_LADDER_129 = [(17, 17, 17), (33, 33, 33), (65, 65, 65), (129, 129, 129)]


class Conf(dict):
    """Tiny stand-in for the pyhocon ConfigTree the reference passes around (config.conf): nested dicts
    addressed with dotted keys, get_float / get_int / get_bool / get_string / get_list / get_config,
    and `in` with dotted keys."""

    def _find(self, key):
        cur = self
        for part in key.split('.'):
            if not isinstance(cur, dict) or not dict.__contains__(cur, part):
                raise KeyError(key)
            cur = dict.__getitem__(cur, part)
        return cur

    def __contains__(self, key):
        try:
            self._find(key)
            return True
        except KeyError:
            return False

    def __getitem__(self, key):
        v = self._find(key)
        return Conf(v) if isinstance(v, dict) and not isinstance(v, Conf) else v

    def get_float(self, k):
        return float(self._find(k))

    def get_int(self, k):
        return int(self._find(k))

    def get_bool(self, k):
        return bool(self._find(k))

    def get_string(self, k):
        return str(self._find(k))

    def get_list(self, k):
        return list(self._find(k))

    def get_config(self, k):
        return Conf(self._find(k))


def reference_config(**overrides):
    """The keys of the reference's config.conf the hot path reads, with its default values
    (config.conf:1-120): train schedule, three loss blocks, network hyper-parameters."""
    loss = dict(color_weight=0.5, grad_weight=0.1, normal_weight=0.1, weighted_normal=True, offset_weight=0.,
                def_regu=dict(weight=2., c=0.5), dct_weight=0.01, sample_pix_num=2048,
                pc_weight=dict(weight=60., mask_weight=1., laplacian_weight=0.1, edge_weight=0., norm_weight=0.01,
                               def_consistent=dict(weight=0.1, c=0.005)))
    level = lambda bs, r, ri: dict(start_epoch=-1, point_render=dict(radius=r, remesh_intersect=ri, batch_size=bs))
    cfg = dict(train=dict(initial_iters=1200, skinner_pose_type=1, learning_rate=1e-4, nepoch=100, sample_pix_num=2048,
                          opt_pose=True, opt_trans=True, opt_camera=False,
                          scheduler=dict(milestones=[60, 80], factor=0.333),
                          coarse=level(3, 0.006, 30), medium=level(2, 0.003, 60), fine=level(1, 0.002, 90)),
               loss_coarse=loss, loss_medium=dict(loss), loss_fine=dict(loss),
               sdf_net=dict(multires=6), mlp_deformer=dict(type='MLPTranslator', condlen=128, multires=6),
               render_net=dict(type='RenderingNetwork_view_norm', condlen=256, multires_p=0, multires_x=0,
                               multires_n=0, multires_v=4))
    cfg.update(overrides)
    return Conf(cfg)


class SyntheticDataset(torch.nn.Module):
    """The two accessors the hot path calls on the reference's dataset (dataset/dataset.py
    get_grad_parameters / get_camera_parameters): per-frame pose / translation / latent codes as
    learnable parameters plus one shared pinhole camera."""

    def __init__(self, n_frames, H, W, seed=5, condlen=128, rendcondlen=0, learn_camera=False):
        super().__init__()
        poses, trans, dcond = make_frame_params(seed, n_frames, condlen)
        self.poses = torch.nn.Parameter(poses)
        self.trans = torch.nn.Parameter(trans)
        self.conds = torch.nn.ParameterList([torch.nn.Parameter(dcond)])
        cam = camera(H, W)
        self.H, self.W = H, W
        self.focals = torch.nn.Parameter(cam["focal"].view(1, 2), requires_grad=learn_camera)
        self.pps = torch.nn.Parameter(cam["pp"].view(1, 2), requires_grad=learn_camera)
        self.register_buffer("Rs", cam["R"].view(1, 3, 3))
        self.Ts = torch.nn.Parameter(cam["T"].view(1, 3), requires_grad=learn_camera)
        self.frame_num = n_frames
        self.video_segmented_index = []

    # ---- the rest of the surface utils.save_model / load_model / getOptNet touch (dataset/dataset.py:26-237)
    @property
    def camera_params(self):
        quat = torch.tensor([0., 0., 0., 1.])       # quat2mat((0,0,0,1)) = diag(-1,-1,1)
        return {'focal_length': self.focals.view(2), 'princeple_points': self.pps.view(2),
                'cam2world_coord_quat': quat, 'world2cam_coord_trans': self.Ts.view(3)}

    def get_batchframe_data(self, name, fids, batchsize):
        """A window of `batchsize` consecutive frames around each id, clamped to the sequence
        (dataset/dataset.py:128-147, single-video branch)."""
        data = getattr(self, name)[:self.frame_num].to(fids.device)
        starts = (fids - batchsize // 2).clamp(min=0, max=max(self.frame_num - batchsize, 0))
        idx = starts.view(-1, 1) + torch.arange(0, batchsize, device=fids.device).view(1, batchsize)
        return data[idx], fids - starts

    def get_grad_parameters(self, frame_ids, device):
        return (self.poses[frame_ids].to(device), self.trans[frame_ids].to(device),
                self.conds[0][frame_ids].to(device), None)

    def get_camera_parameters(self, n, device):
        return (self.focals.expand(n, 2).to(device), self.pps.expand(n, 2).to(device),
                self.Rs.expand(n, 3, 3).to(device), self.Ts.expand(n, 3).to(device), self.H, self.W)


class _LazyFrames:
    """Frame i of a seeded smooth sequence, made when write_sequence asks for it (a 600-frame 1080p sequence would not
    fit in host memory as float arrays)."""

    def __init__(self, F, H, W, seed, kind):
        self.F, self.H, self.W, self.kind = F, H, W, kind
        rs = np.random.RandomState(seed)
        self.freq = rs.uniform(0.5, 3.0, (3, 2))
        self.phase = rs.uniform(0, 2 * np.pi, (F, 3))

    def __len__(self):
        return self.F

    def __getitem__(self, i):
        y = np.linspace(-1, 1, self.H, dtype=np.float32)[:, None]
        x = np.linspace(-1, 1, self.W, dtype=np.float32)[None, :]
        if self.kind == "mask":   # an ellipse drifting with the frame index
            cx = 0.3 * np.sin(0.2 * i)
            return (((x - cx) / 0.45) ** 2 + (y / 0.8) ** 2 < 1).astype(np.float32)
        ch = [np.sin(np.pi * (self.freq[c, 0] * x + self.freq[c, 1] * y) + self.phase[i, c]) for c in range(3)]
        out = np.stack(np.broadcast_arrays(*ch), -1).astype(np.float32)
        if self.kind == "normal":
            out = out / np.maximum(np.linalg.norm(out, axis=-1, keepdims=True), 1e-6)
        return 0.9 * out if self.kind == "img" else out


def write_frame_sequence(root, F, H, W, seed=0, normals=True, image_ext=".png"):
    """A seeded sequence of F smooth H x W frames in the on-disk layout of dataset.SceneDataset (written by
    dataset.write_sequence; image_ext='.jpg' re-encodes the images as JPEG).  -> root"""
    import os
    import cv2
    from dataset import write_sequence
    poses, trans, _ = make_frame_params(seed, F)
    cam = dict(fx=float(W), fy=float(W), cx=W / 2.0, cy=H / 2.0, quat=[0., 0., 0., 1.], T=[0., 0., 2.5])
    write_sequence(root, _LazyFrames(F, H, W, seed, "img"), _LazyFrames(F, H, W, seed + 1, "mask"), poses.numpy(),
                   trans.numpy(), np.zeros(10, np.float32), cam,
                   normals=_LazyFrames(F, H, W, seed + 2, "normal") if normals else None)
    if image_ext != ".png":
        for i in range(F):
            p = os.path.join(root, "imgs", "%06d.png" % i)
            cv2.imwrite(p[:-4] + image_ext, cv2.imread(p))
            os.remove(p)
    return root
