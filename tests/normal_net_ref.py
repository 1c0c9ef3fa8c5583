"""Float64 twin of the normal-map step (selfreconcode_b200/normals.py, csrc/normal_net.cu).

  GlobalGenerator: a torch restatement of pix2pixHD's generator that PIFuHD's front-normal net is
      (define_G(3, 3, 64, "global", 4, 9, 1, 3, "instance")): ReflectionPad(3) + Conv 7x7 + IN + ReLU, n_down x
      [Conv k3 s2 p1 + IN + ReLU], n_blocks x ResnetBlock (pad, conv, IN, ReLU, pad, conv, IN, + input), n_down x
      [ConvTranspose k3 s2 p1 op1 + IN + ReLU], ReflectionPad(3) + Conv 7x7 + Tanh; InstanceNorm2d(affine=False).
      Its module names give the state_dict keys PIFuHD's checkpoint holds under 'netG.netF.'.
  unwarp_quantise: numpy restatement of generate_normals.py:149-165 (grid_sample back onto the frame, |n| < 1e-4 and
      background -> 0, (n*0.5 + 0.5)[::-1]*255) in float64, before the uint8 truncation.
"""
import numpy as np
import torch
from torch import nn


class ResnetBlock(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.conv_block = nn.Sequential(nn.ReflectionPad2d(1), nn.Conv2d(dim, dim, 3), nn.InstanceNorm2d(dim),
                                        nn.ReLU(True), nn.ReflectionPad2d(1), nn.Conv2d(dim, dim, 3),
                                        nn.InstanceNorm2d(dim))

    def forward(self, x):
        return x + self.conv_block(x)


class GlobalGenerator(nn.Module):
    def __init__(self, in_nc=3, out_nc=3, ngf=64, n_down=4, n_blocks=9):
        super().__init__()
        m = [nn.ReflectionPad2d(3), nn.Conv2d(in_nc, ngf, 7), nn.InstanceNorm2d(ngf), nn.ReLU(True)]
        for i in range(n_down):
            c = ngf * 2 ** i
            m += [nn.Conv2d(c, 2 * c, 3, stride=2, padding=1), nn.InstanceNorm2d(2 * c), nn.ReLU(True)]
        m += [ResnetBlock(ngf * 2 ** n_down) for _ in range(n_blocks)]
        for i in range(n_down):
            c = ngf * 2 ** (n_down - i)
            m += [nn.ConvTranspose2d(c, c // 2, 3, stride=2, padding=1, output_padding=1), nn.InstanceNorm2d(c // 2),
                  nn.ReLU(True)]
        m += [nn.ReflectionPad2d(3), nn.Conv2d(ngf, out_nc, 7), nn.Tanh()]
        self.model = nn.Sequential(*m)

    def forward(self, x):
        return self.model(x)


SMALL = dict(in_nc=3, out_nc=3, ngf=8, n_down=2, n_blocks=2)


def seeded_net(seed=0, **arch):
    """GlobalGenerator with torch's default initialisation under a fixed seed (float64, CPU)."""
    torch.manual_seed(seed)
    return GlobalGenerator(**arch).double().eval()


def forward64(net, x, device="cpu"):
    """x [B,3,S,S] -> the twin's output in float64 on `device` (the net is moved there)."""
    net = net.to(device)
    with torch.no_grad():
        return net(torch.as_tensor(x).to(device=device, dtype=torch.float64))


def unwarp_values(nml, rect, H, W):
    """nml [3,S,S] (any float) sampled onto H x W through rect [x, y, w, h] as grid_sample(bilinear, zeros,
    align_corners=True) in float64 -> [H,W,3]."""
    nml = np.asarray(nml, np.float64)
    S = nml.shape[-1]
    x, y, w, h = [float(v) for v in rect]
    cols, rows = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    ix = (2.0 * (cols - x) / w - 1.0 + 1.0) * (S - 1) / 2.0
    iy = (2.0 * (rows - y) / h - 1.0 + 1.0) * (S - 1) / 2.0
    x0, y0 = np.floor(ix), np.floor(iy)
    fx, fy = ix - x0, iy - y0
    out = np.zeros((H, W, 3))
    for dy, wy in ((0, 1 - fy), (1, fy)):
        for dx, wx in ((0, 1 - fx), (1, fx)):
            xi, yi = (x0 + dx).astype(np.int64), (y0 + dy).astype(np.int64)
            ok = (xi >= 0) & (xi < S) & (yi >= 0) & (yi < S)
            v = nml[:, np.clip(yi, 0, S - 1), np.clip(xi, 0, S - 1)].transpose(1, 2, 0)
            out += np.where(ok[..., None], v, 0.0) * (wx * wy)[..., None]
    return out


def unwarp_quantise(nml, rect, fg, H, W):
    """generate_normals.py:149-165 in float64, before astype(uint8): -> (values [H,W,3] BGR, zeroed bool [H,W])."""
    n = unwarp_values(nml, rect, H, W)
    zero = np.linalg.norm(n, axis=-1) < 1e-4
    if fg is not None:
        zero |= ~np.asarray(fg, bool)
    v = (n * 0.5 + 0.5)[:, :, ::-1] * 255.0
    v[zero] = 0.0
    return v, zero


STANDIN_B = (0.0625, -0.125, 0.03125)


def standin(x):
    """The stand-in network oracle/make_golden_normals.py gives the unmodified script: x float32 [3,S,S] -> channel o
    = round((0.5 x[o] + 0.25 x[o+1] - 0.125 x[o+2] + b[o]) * 1024) / 1024, left to right in float32 (bit-exact)."""
    f = np.float32
    x = np.asarray(x, f)
    out = []
    for o in range(3):
        t = x[o] * f(0.5)
        t = t + x[(o + 1) % 3] * f(0.25)
        t = t - x[(o + 2) % 3] * f(0.125)
        t = t + f(STANDIN_B[o])
        out.append(np.round(t * f(1024.0)) / f(1024.0))
    return np.stack(out).astype(f)


def sha256(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def unwarp_f32(nml, rect, fg, H, W):
    """generate_normals.py:149-165 in the float32 order of torch's CPU grid sampler and the script's numpy
    expressions (the order csrc/normal_net.cu follows) -> uint8 BGR [H,W,3]."""
    f = np.float32
    nml = np.asarray(nml, f)
    S = nml.shape[-1]
    x, y, w, h = [f(v) for v in rect]
    cols, rows = np.meshgrid(np.arange(W, dtype=f), np.arange(H, dtype=f))
    gx = (f(2) * (cols - x)) / w - f(1)
    gy = (f(2) * (rows - y)) / h - f(1)
    scale = f(S - 1) / f(2)
    ix, iy = (gx + f(1)) * scale, (gy + f(1)) * scale
    x0, y0 = np.floor(ix), np.floor(iy)
    we, wn = ix - x0, iy - y0
    e, s = f(1) - we, f(1) - wn
    xi, yi = x0.astype(np.int64), y0.astype(np.int64)

    def corner(dy, dx):
        xx, yy = xi + dx, yi + dy
        ok = (xx >= 0) & (xx < S) & (yy >= 0) & (yy < S)
        v = nml[:, np.clip(yy, 0, S - 1), np.clip(xx, 0, S - 1)]
        return np.where(ok[None], v, f(0))
    v = corner(0, 0) * (s * e) + corner(0, 1) * (s * we)
    v = v + corner(1, 0) * (wn * e)
    v = v + corner(1, 1) * (wn * we)
    sq = v[0] * v[0]
    sq = sq + v[1] * v[1]
    sq = sq + v[2] * v[2]
    zero = np.sqrt(sq) < f(1e-4)
    if fg is not None:
        zero |= ~np.asarray(fg, bool)
    q = (np.transpose(v, (1, 2, 0)) * f(0.5) + f(0.5))[:, :, ::-1] * f(255.0)
    q[zero] = 0
    return q.astype(np.uint8)
