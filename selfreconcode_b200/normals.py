"""Normal maps of a sequence from PIFuHD's front-normal network, on the device (generate_normals.py of the reference).

The reference runs `lib.networks.define_G(3, 3, 64, "global", 4, 9, 1, 3, "instance")` from a PIFuHD checkout on
512 x 512 crops whose boxes a Lightweight OpenPose checkout wrote (generate_boxs.py).  Here the network is pix2pixHD's
GlobalGenerator restated on this library's kernels (csrc/normal_net.cu + the tensor-core layer kernel), the weights
are read from the same checkpoint, and frames without a box file get one from their mask:

    python -m selfreconcode_b200.normals --imgpath <seq>/imgs [--weights checkpoints/pifuhd.pt] [--gid 0]

writes <seq>/normals/<fold>/<stem>.png (uint8 BGR, what SceneDataset reads back) and video.avi per folder.

Host steps (image read, mask, RGBA composite, crop, 512 x 512 resize, normalisation) run with cv2 / numpy exactly as
the script does, so the network input is the reference's bit for bit; decode and encode run on a thread pool.

Differences from the reference, all deliberate:
  * a frame without `<stem>_rect.txt` is processed (the reference skips it) with a square box from its mask: the
    bounding box [x0, x1] x [y0, y1] of the foreground, centre ((x0 + x1) // 2, (y0 + y1) // 2), radius
    int(0.57 * max(w, h)) (at least 1).  0.57 is generate_boxs.py:49-54's 0.65 x keypoint extent with keypoints
    spanning about 0.87 of a standing person's silhouette -- a heuristic nobody has compared with OpenPose boxes.
    No mask, or an empty one: generate_boxs.py:60-62's image centre with radius max(W, H) // 2;
  * frames of the same size run through the network in batches (instance norm is per sample, so a frame's result
    does not depend on its batch);
  * grid_sample's coordinates use true division, as torch's CPU path does (its CUDA path multiplies by 1/w).
"""
import argparse
import os
import os.path as osp
from collections import OrderedDict
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib, ops

CROP = 512                      # generate_normals.py:97
IMG_EXTS = ('png', 'jpeg', 'jpg', 'PNG', 'JPG', 'JPEG')
PIFUHD_ARCH = dict(in_nc=3, out_nc=3, ngf=64, n_down=4, n_blocks=9)   # define_G(3, 3, 64, "global", 4, 9, ...)
PREFIX = 'netG.netF.'
MAX_BATCH = 16
WORKSPACE_BYTES = 1 << 30       # im2col operand of one row chunk


# ---- network layout --------------------------------------------------------------------------------------------
def layer_keys(in_nc=3, out_nc=3, ngf=64, n_down=4, n_blocks=9):
    """state_dict keys and shapes of GlobalGenerator(in_nc, out_nc, ngf, n_down, n_blocks) with instance norm (no
    affine parameters): the indices of its nn.Sequential `model`."""
    keys = OrderedDict()

    def conv(name, shape):
        keys[name + '.weight'] = tuple(shape)
        keys[name + '.bias'] = (shape[1] if name in ups else shape[0],)
    ups = set()
    conv('model.1', (ngf, in_nc, 7, 7))                                  # ReflectionPad(3), Conv 7x7, IN, ReLU
    i = 4
    for d in range(n_down):                                              # Conv k3 s2 p1, IN, ReLU
        conv('model.%d' % i, (ngf * 2 ** (d + 1), ngf * 2 ** d, 3, 3))
        i += 3
    c = ngf * 2 ** n_down
    for _ in range(n_blocks):                                            # ResnetBlock: pad, conv, IN, ReLU, pad, conv, IN
        conv('model.%d.conv_block.1' % i, (c, c, 3, 3))
        conv('model.%d.conv_block.5' % i, (c, c, 3, 3))
        i += 1
    for u in range(n_down):                                              # ConvTranspose k3 s2 p1 op1, IN, ReLU
        ci = ngf * 2 ** (n_down - u)
        ups.add('model.%d' % i)
        conv('model.%d' % i, (ci, ci // 2, 3, 3))
        i += 3
    conv('model.%d' % (i + 1), (out_nc, ngf, 7, 7))                      # ReflectionPad(3), Conv 7x7, Tanh
    return keys


def _shape(v):
    return tuple(int(s) for s in v.shape)


def architecture(sd):
    """(in_nc, out_nc, ngf, n_down, n_blocks) read from a GlobalGenerator state dict's keys and shapes; then the
    whole key set is checked like load_state_dict(strict=True): a missing, unexpected or misshapen key raises
    KeyError / ValueError naming it."""
    if 'model.1.weight' not in sd:
        raise KeyError("front-normal weights: missing key 'model.1.weight' (not a GlobalGenerator state dict)")
    ngf, in_nc = _shape(sd['model.1.weight'])[:2]
    n_down, i, c = 0, 4, ngf
    while 'model.%d.weight' % i in sd and _shape(sd['model.%d.weight' % i]) == (2 * c, c, 3, 3):
        n_down, i, c = n_down + 1, i + 3, 2 * c
    n_blocks = 0
    while 'model.%d.conv_block.1.weight' % i in sd:
        n_blocks, i = n_blocks + 1, i + 1
    last = 'model.%d.weight' % (i + 3 * n_down + 1)
    out_nc = _shape(sd[last])[0] if last in sd and len(sd[last].shape) == 4 else 3
    arch = dict(in_nc=in_nc, out_nc=out_nc, ngf=ngf, n_down=n_down, n_blocks=n_blocks)
    want = layer_keys(**arch)
    for k in want:
        if k not in sd:
            raise KeyError("front-normal weights: missing key %r (layout read as %s)" % (k, arch))
    for k in sd:
        if k not in want:
            raise KeyError("front-normal weights: unexpected key %r (layout read as %s)" % (k, arch))
    for k, sh in want.items():
        if _shape(sd[k]) != sh:
            raise ValueError("front-normal weights: %r has shape %s, expected %s (layout read as %s)"
                             % (k, _shape(sd[k]), sh, arch))
    return arch


def read_state_dict(path_or_state_dict):
    """generate_normals.py:118-121: torch.load(path)['model_state_dict'], the keys under 'netG.netF.' with the prefix
    stripped; a bare state dict (with or without the prefix) is taken as it is."""
    sd = path_or_state_dict
    if isinstance(sd, (str, os.PathLike)):
        sd = torch.load(sd, map_location='cpu', weights_only=False)
    if 'model_state_dict' in sd:
        sd = sd['model_state_dict']
    if any(k.startswith(PREFIX) for k in sd):
        sd = OrderedDict((k[len(PREFIX):], v) for k, v in sd.items() if k.startswith(PREFIX))
    return sd


class FrontNormalNet:
    """GlobalGenerator forward on the device: `net(x)` with x CUDA fp32 [B,in_nc,S,S] in [-1, 1] -> [B,out_nc,S,S]
    (tanh), on the current stream, no autograd.  Every conv is csrc/normal_net.cu's im2col pack + sr_tc_linear;
    instance norm is sr_instance_norm_stats / _apply."""

    def __init__(self, sd, device):
        self.arch = architecture(sd)
        self.device = torch.device(device)
        a = self.arch
        t = lambda k: sd[k].to(self.device)
        conv = lambda name, **kw: ops.TcConv(t(name + '.weight'), t(name + '.bias'), **kw)
        with torch.cuda.device(self.device):
            self.first = conv('model.1', pad=3, pad_mode='reflect')
            self.down = [conv('model.%d' % (4 + 3 * d), stride=2, pad=1) for d in range(a['n_down'])]
            r0 = 4 + 3 * a['n_down']
            self.blocks = [(conv('model.%d.conv_block.1' % (r0 + j), pad=1, pad_mode='reflect'),
                            conv('model.%d.conv_block.5' % (r0 + j), pad=1, pad_mode='reflect'))
                           for j in range(a['n_blocks'])]
            u0 = r0 + a['n_blocks']
            self.up = [conv('model.%d' % (u0 + 3 * u), stride=2, pad=1, transposed=True, output_padding=1)
                       for u in range(a['n_down'])]
            self.last = conv('model.%d' % (u0 + 3 * a['n_down'] + 1), pad=3, pad_mode='reflect')
            self.workspace = torch.empty((WORKSPACE_BYTES,), dtype=torch.uint8, device=self.device)
        self.chunk_rows = None      # row chunks of the im2col operand; None = as many rows as the workspace holds

    def bytes_per_frame(self, S):
        """device memory one frame of side S needs beyond the weights and workspace (the widest layer's input, output
        and instance-norm input, fp32, and the net input / output)."""
        widest = max(S * S * self.arch['ngf'], (S >> self.arch['n_down']) ** 2 * self.arch['ngf'] << self.arch['n_down'])
        return 4 * (3 * widest + 2 * S * S * (self.arch['in_nc'] + self.arch['out_nc']))

    def _conv_in(self, x, conv, relu=True, residual=None):
        y = ops.conv2d(x, conv, self.workspace, chunk_rows=self.chunk_rows)
        mean, rstd = ops.instance_norm_stats(y)
        return ops.instance_norm_apply(y, mean, rstd, residual=residual, relu=relu, out=y)

    def forward_cl(self, x):
        """channels-last: x fp32 [B,S,S,in_nc] -> tanh output fp32 [B,S,S,out_nc]."""
        with torch.no_grad(), torch.cuda.device(self.device):
            h = self._conv_in(x.contiguous(), self.first)
            for c in self.down:
                h = self._conv_in(h, c)
            for c1, c2 in self.blocks:
                h = self._conv_in(self._conv_in(h, c1), c2, relu=False, residual=h)
            for c in self.up:
                h = self._conv_in(h, c)
            return ops.conv2d(h, self.last, self.workspace, act=_lib.SR_ACT_TANH, chunk_rows=self.chunk_rows)

    def __call__(self, x):
        if not x.is_cuda or x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != self.arch['in_nc']:
            raise ValueError("FrontNormalNet: expected a CUDA fp32 [B,%d,S,S] tensor" % self.arch['in_nc'])
        with torch.no_grad():
            return self.forward_cl(x.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2).contiguous()


def load_front_net(path_or_state_dict, device):
    """PIFuHD's front-normal net from `checkpoints/pifuhd.pt` (or a state dict) on `device` -> FrontNormalNet."""
    return FrontNormalNet(read_state_dict(path_or_state_dict), device)


# ---- host steps (generate_normals.py:21-102) --------------------------------------------------------------------
def crop_image(img, rect):
    """generate_normals.py:21-38: the rect [x, y, w, h] of img, zero outside the image."""
    import cv2
    x, y, w, h = rect
    left = abs(x) if x < 0 else 0
    top = abs(y) if y < 0 else 0
    right = abs(img.shape[1] - (x + w)) if x + w >= img.shape[1] else 0
    bottom = abs(img.shape[0] - (y + h)) if y + h >= img.shape[0] else 0
    padded = cv2.copyMakeBorder(img, top, bottom, left, right, cv2.BORDER_CONSTANT, value=[0] * img.shape[2])
    return padded[y + top:y + top + h, x + left:x + left + w, :]


def choose_rect(rects):
    """generate_normals.py:81-95: one row -> it; several -> the first with the largest (w + h) // 2 (strict <, so the
    last row when none is positive)."""
    rects = np.asarray(rects, dtype=np.int32)
    if rects.ndim == 1:
        return rects.tolist()
    max_len, pid = 0, -1
    for ind, r in enumerate(rects):
        cur = (r[-2] + r[-1]) // 2
        if max_len < cur:
            max_len, pid = cur, ind
    return rects[pid].tolist()


def mask_box(fg, H, W):
    """Square crop box [x, y, 2r, 2r] from a foreground mask (bool [H,W] or None); see the module docstring."""
    if fg is None or not fg.any():
        cx, cy, r = W // 2, H // 2, max(W // 2, H // 2)
    else:
        ys, xs = np.nonzero(fg.any(1))[0], np.nonzero(fg.any(0))[0]
        x0, x1, y0, y1 = int(xs[0]), int(xs[-1]), int(ys[0]), int(ys[-1])
        cx, cy = (x0 + x1) // 2, (y0 + y1) // 2
        r = max(1, int(0.57 * max(x1 - x0 + 1, y1 - y0 + 1)))
    return [cx - r, cy - r, 2 * r, 2 * r]


def rect_path(img_path):
    ext = img_path.split('.')[-1]
    return img_path.replace('.%s' % ext, '_rect.txt')          # generate_normals.py:58


def mask_path(img_path):
    return img_path.replace('/imgs/', '/masks/')[:-3] + 'png'   # generate_normals.py:59


def list_frames(root):
    """generate_normals.py:45-46 without the rect-file filter: the image files of `root` sorted by int(stem)."""
    files = [osp.join(root, f) for f in os.listdir(root) if f.split('.')[-1] in IMG_EXTS]
    files.sort(key=lambda p: int(osp.basename(p).split('.')[0]))
    return files


def list_folds(imgpath):
    """generate_normals.py:128-130: the digit-named subfolders of imgpath, or '.'."""
    cids = sorted((d for d in os.listdir(imgpath) if osp.isdir(osp.join(imgpath, d)) and d.isdigit()), key=int)
    return cids if cids else ['.']


def prepare_frame(img_path):
    """generate_normals.py:56-102 for one image -> dict(name, x fp32 [3,512,512] (normalised RGB), fg bool [H,W] or
    None, H, W, rect [x, y, w, h], rect_from ('file' | 'mask' | 'centre'))."""
    import cv2
    im = cv2.imread(img_path, cv2.IMREAD_UNCHANGED)
    if im is None:
        raise ValueError("%s: unreadable image" % img_path)
    if im.ndim == 2:
        im = im[:, :, None]
    mp = mask_path(img_path)
    fg = None
    if osp.isfile(mp):
        mask = cv2.imread(mp)
        fg = (mask > 0).all(-1)
        im[~fg] = np.zeros(im.shape[-1], dtype=im.dtype)
    H, W = im.shape[:2]
    if im.shape[2] == 4:                                         # :73-77, composite onto 0.5 grey
        im = im / 255.0
        im[:, :, :3] /= im[:, :, 3:] + 1e-8
        im = im[:, :, 3:] * im[:, :, :3] + 0.5 * (1.0 - im[:, :, 3:])
        im = (255.0 * im).astype(np.uint8)
    rp = rect_path(img_path)
    rect = None
    if osp.isfile(rp):
        rects = np.loadtxt(rp, dtype=np.int32)
        if rects.size:
            rect, src = choose_rect(rects), 'file'
    if rect is None:
        rect = mask_box(fg, H, W)
        src = 'mask' if fg is not None and fg.any() else 'centre'
    im512 = cv2.resize(crop_image(im, rect), (CROP, CROP))
    # PIL convert('RGB') + ToTensor + Normalize(0.5, 0.5): (u8 / 255 - 0.5) / 0.5 in float32
    rgb = np.ascontiguousarray(im512[:, :, 2::-1] if im512.ndim == 3 else np.repeat(im512[:, :, None], 3, -1))
    x = (rgb.astype(np.float32) / np.float32(255.) - np.float32(0.5)) / np.float32(0.5)
    return dict(name=osp.splitext(osp.basename(img_path))[0], x=np.ascontiguousarray(x.transpose(2, 0, 1)), fg=fg,
                H=H, W=W, rect=[int(v) for v in rect], rect_from=src)


def normals_on_device(net, frames, device):
    """Network + sr_normal_unwarp for frames of one size (prepare_frame dicts) -> uint8 BGR [B,H,W,3] on the host."""
    H, W = frames[0]['H'], frames[0]['W']
    x = torch.from_numpy(np.stack([f['x'] for f in frames])).to(device, non_blocking=False)
    nml = net.forward_cl(x.permute(0, 2, 3, 1).contiguous())
    boxes = torch.tensor([f['rect'] for f in frames], dtype=torch.float32, device=device)
    fg = None
    if any(f['fg'] is not None for f in frames):
        fg = torch.from_numpy(np.stack([f['fg'] if f['fg'] is not None else np.ones((H, W), np.bool_)
                                        for f in frames]).view(np.uint8)).to(device)
    with torch.cuda.device(device):
        return ops.normal_unwarp(nml, boxes, fg, H, W).cpu().numpy()


def batch_size_for(net, S, device):
    """MAX_BATCH frames, fewer when the device's free memory (half of it) does not hold them."""
    free = torch.cuda.mem_get_info(device)[0]
    return int(max(1, min(MAX_BATCH, (free // 2) // net.bytes_per_frame(S))))


def generate_normals(imgpath, weights='checkpoints/pifuhd.pt', device=0):
    """generate_normals.py's loop: for each folder of imgpath (digit-named subfolders, or imgpath itself) writes
    imgpath/../normals/<fold>/<stem>.png for every image, and video.avi (MJPG, 30 fps, the first frame's size).
    -> {output png path: 'file' | 'mask' | 'centre' (where its crop box came from)}."""
    import cv2
    device = torch.device('cuda', device) if isinstance(device, int) else torch.device(device)
    net = load_front_net(weights, device)
    B = batch_size_for(net, CROP, device)
    written = {}
    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as pool:
        for fold in list_folds(imgpath):
            save_root = osp.normpath(osp.join(imgpath, osp.pardir, 'normals', fold))
            os.makedirs(save_root, exist_ok=True)
            print(save_root)
            files = list_frames(osp.normpath(osp.join(imgpath, fold)))
            ahead = [pool.submit(prepare_frame, p) for p in files[:2 * B]]   # decoded ahead of the device
            writer, writes, pending = None, [], []

            def flush(group):
                nonlocal writer
                out = normals_on_device(net, group, device)
                for f, n in zip(group, out):
                    if writer is None:
                        writer = cv2.VideoWriter(osp.join(save_root, 'video.avi'), cv2.VideoWriter.fourcc(*'MJPG'),
                                                 30., (f['W'], f['H']))
                    dst = osp.join(save_root, f['name'] + '.png')
                    writes.append(pool.submit(cv2.imwrite, dst, n))
                    writer.write(n)
                    written[dst] = f['rect_from']
            for i in range(len(files)):
                f = ahead[i].result()
                ahead[i] = None
                if i + 2 * B < len(files):
                    ahead.append(pool.submit(prepare_frame, files[i + 2 * B]))
                if pending and ((f['H'], f['W']) != (pending[0]['H'], pending[0]['W']) or len(pending) == B):
                    flush(pending)
                    pending = []
                pending.append(f)
            if pending:
                flush(pending)
            for w in writes:
                if not w.result():
                    raise IOError("normal map not written")
            if writer is not None:
                writer.release()
    print('done.')
    return written


def main(argv=None):
    p = argparse.ArgumentParser(description='front normal maps of a sequence (generate_normals.py)')
    p.add_argument('--gid', default=0, type=int, metavar='ID', help='gpu id')
    p.add_argument('--imgpath', required=True, metavar='M', help='the sequence\'s imgs folder')
    p.add_argument('--weights', default='checkpoints/pifuhd.pt', help='PIFuHD checkpoint (model_state_dict)')
    args = p.parse_args(argv)
    generate_normals(args.imgpath, args.weights, args.gid)


if __name__ == '__main__':
    main()
