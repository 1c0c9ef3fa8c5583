"""GPU: the front-normal network and normal-map step on the device (csrc/normal_net.cu, ops.TcConv / conv2d,
selfreconcode_b200/normals.py) against float64: each conv kind through the im2col pack + the tensor-core layer kernel
at its tiling edges, instance norm, determinism and batch independence, the whole network against the float64 twin
(tests/normal_net_ref.py) at a small shape and at PIFuHD's, the unwarp against the PNGs the unmodified script wrote
(tests/golden/normals_io.npz), and generate_normals end to end into the training loader's frame store."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import normal_net_ref as R
from helpers import dropin, golden

pytestmark = pytest.mark.gpu

WS = 64 << 20


def _ops():
    from selfreconcode_b200 import _lib, ops
    _lib.load()
    return ops


# (B, H, W, Cin, Cout, k, stride, pad, mode, transposed, chunk_rows, act)
CONVS = {
    "7x7-reflect-cin3": (2, 37, 41, 3, 64, 7, 1, 3, "reflect", False, None, 0),
    "7x7-reflect-cin64-n3-tanh": (1, 40, 36, 64, 3, 7, 1, 3, "reflect", False, 384, 3),
    "3x3-s2-zero-n128": (3, 33, 30, 64, 128, 3, 2, 1, "zeros", False, None, 0),
    "3x3-s2-zero-chunks": (2, 31, 29, 128, 256, 3, 2, 1, "zeros", False, 128, 0),
    "3x3-reflect-n1024": (2, 8, 9, 1024, 1024, 3, 1, 1, "reflect", False, None, 0),
    "3x3-reflect-cin5-chunks": (2, 19, 23, 5, 64, 3, 1, 1, "reflect", False, 256, 0),
    "convT-s2-op1": (2, 9, 7, 256, 128, 3, 2, 1, "zeros", True, None, 0),
    "convT-s2-op1-n64-chunks": (1, 16, 13, 128, 64, 3, 2, 1, "zeros", True, 128, 0),
}


@pytest.mark.parametrize("name", list(CONVS))
def test_conv_kinds_vs_float64(name, cuda_dev):
    ops = _ops()
    B, H, W, Cin, Cout, k, s, p, mode, tr, chunk, act = CONVS[name]
    g = torch.Generator().manual_seed(len(name))
    x = torch.randn(B, Cin, H, W, generator=g)
    if tr:
        w = (torch.rand(Cin, Cout, k, k, generator=g) * 2 - 1) / (Cin * k * k) ** 0.5
    else:
        w = (torch.rand(Cout, Cin, k, k, generator=g) * 2 - 1) / (Cin * k * k) ** 0.5
    b = torch.rand(Cout, generator=g) - 0.5
    xd, wd, bd = x.double(), w.double(), b.double()
    if tr:
        ref = F.conv_transpose2d(xd, wd, bd, stride=s, padding=p, output_padding=1)
    elif mode == "reflect":
        ref = F.conv2d(F.pad(xd, (p,) * 4, mode="reflect"), wd, bd, stride=s)
    else:
        ref = F.conv2d(xd, wd, bd, stride=s, padding=p)
    # sum of |products| per output: the split-bf16 GEMM's error grows with it and with K (truncating accumulation)
    xa, wa = xd.abs(), wd.abs()
    if tr:
        mag = F.conv_transpose2d(xa, wa, None, stride=s, padding=p, output_padding=1)
    elif mode == "reflect":
        mag = F.conv2d(F.pad(xa, (p,) * 4, mode="reflect"), wa, None, stride=s)
    else:
        mag = F.conv2d(xa, wa, None, stride=s, padding=p)
    if act == 3:
        ref = torch.tanh(ref)
    conv = ops.TcConv(w.to(cuda_dev), b.to(cuda_dev), stride=s, pad=p, pad_mode=mode, transposed=tr,
                      output_padding=1 if tr else 0)
    ws = torch.empty(WS, dtype=torch.uint8, device=cuda_dev)
    out = ops.conv2d(x.permute(0, 2, 3, 1).contiguous().to(cuda_dev), conv, ws, act=act, chunk_rows=chunk)
    assert out.shape == (B,) + tuple(ref.shape[2:]) + (Cout,)
    got = out.permute(0, 3, 1, 2).double().cpu()
    err = float((got - ref).abs().max())
    scale = float(mag.max()) + 1.0
    print("%s: M %d, K %d, N %d: max |d| %.3g (max sum |x w| + |b| <= %.3g)" % (name, out.numel() // Cout, Cin * k * k,
                                                                               Cout, err, scale))
    assert err <= 2.0 ** -16 * scale, name
    if chunk is not None:                           # chunks cut inside a sample: the same bits as one chunk
        one = ops.conv2d(x.permute(0, 2, 3, 1).contiguous().to(cuda_dev), conv,
                         torch.empty(1 << 30, dtype=torch.uint8, device=cuda_dev), act=act)
        assert torch.equal(one, out), name


@pytest.mark.parametrize("relu,residual", [(True, False), (False, True), (False, False)])
def test_instance_norm_vs_float64(relu, residual, cuda_dev):
    ops = _ops()
    g = torch.Generator().manual_seed(7)
    B, H, W, C = 3, 45, 37, 96                     # H*W = 1665: slices of 512 with a partial last one
    y = torch.randn(B, H, W, C, generator=g) * (1 + torch.rand(C, generator=g) * 3) + torch.randn(C, generator=g) * 4
    r = torch.randn(B, H, W, C, generator=g)
    yd = y.double()
    mu = yd.mean(dim=(1, 2))
    var = yd.var(dim=(1, 2), unbiased=False)
    mean, rstd = ops.instance_norm_stats(y.to(cuda_dev))
    assert float((mean.double().cpu() - mu).abs().max()) < 1e-6 * float(mu.abs().max() + 1)
    assert float(((rstd.double().cpu() - 1 / torch.sqrt(var + 1e-5)) * torch.sqrt(var + 1e-5)).abs().max()) < 1e-6
    ref = (yd - mu[:, None, None]) / torch.sqrt(var[:, None, None] + 1e-5)
    if relu:
        ref = ref.clamp_min(0)
    if residual:
        ref = ref + r.double()
    out = ops.instance_norm_apply(y.to(cuda_dev), mean, rstd, residual=r.to(cuda_dev) if residual else None,
                                  relu=relu)
    assert float((out.double().cpu() - ref).abs().max()) < 1e-5
    # torch's own fp64 InstanceNorm2d agrees with the statistics restated above
    tin = F.instance_norm(yd.permute(0, 3, 1, 2), eps=1e-5).permute(0, 2, 3, 1)
    assert float((tin - (yd - mu[:, None, None]) / torch.sqrt(var[:, None, None] + 1e-5)).abs().max()) < 1e-10


def _smooth_input(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    lo = torch.rand(B, 3, 12, 12, generator=g) * 2 - 1
    return F.interpolate(lo, size=(S, S), mode="bilinear", align_corners=False).clamp(-1, 1).contiguous()


def _net(arch, seed, dev):
    from selfreconcode_b200 import normals as N
    twin = R.seeded_net(seed, **arch)
    return twin, N.load_front_net({k: v.float() for k, v in twin.state_dict().items()}, dev)


def test_determinism_and_batch_independence(cuda_dev):
    _, net = _net(R.SMALL, 1, cuda_dev)
    x = _smooth_input(17, 64, 2).to(cuda_dev)
    a = net(x)
    b = net(x)
    assert torch.equal(a, b)
    one = net(x[5:6].contiguous())
    assert torch.equal(one[0], a[5])
    net.chunk_rows = 384                            # chunks cut inside samples change no bit
    assert torch.equal(net(x), a)


def _compare(net, twin, x, dev, label):
    got = net(x.to(dev)).double().cpu()
    ref = torch.cat([R.forward64(twin, x[i:i + 1], dev).cpu() for i in range(x.shape[0])])
    d = (got - ref).abs()
    mx, p999 = float(d.max()), float(torch.quantile(d.reshape(-1)[::7].float(), 0.999))
    print("%s: max |d| %.3g, 99.9th pct %.3g, |out| mean %.3f" % (label, mx, p999, float(ref.abs().mean())))
    assert mx <= 1e-3, label
    return mx


def test_network_small_vs_twin(cuda_dev):
    twin, net = _net(R.SMALL, 3, cuda_dev)
    _compare(net, twin, _smooth_input(3, 64, 4), cuda_dev, "ngf 8, 2 down, 2 blocks, 64x64, B 3")


@pytest.mark.parametrize("B", [2, 17])
def test_network_pifuhd_shape_vs_twin(B, cuda_dev):
    from selfreconcode_b200 import normals as N
    twin, net = _net(N.PIFUHD_ARCH, 0, cuda_dev)
    _compare(net, twin, _smooth_input(B, 512, 5 + B), cuda_dev, "PIFuHD shape 512x512, B %d" % B)


def _golden_tree(tmp_path):
    g = golden("normals_io.npz")
    for k in g.files:
        if k.startswith("files/"):
            p = os.path.join(str(tmp_path), k[6:])
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as f:
                f.write(g[k].tobytes())
    return g


def test_unwarp_bitwise_vs_script(tmp_path, cuda_dev):
    from selfreconcode_b200 import normals as N
    ops = _ops()
    g = _golden_tree(tmp_path)
    for key in g["frames"]:
        lay, fold, stem = key.split("|")
        root = os.path.normpath(os.path.join(str(tmp_path), lay, "imgs", fold))
        path = [p for p in N.list_frames(root) if os.path.basename(p).split(".")[0] == stem][0]
        f = N.prepare_frame(path)
        y = R.standin(f["x"])
        assert R.sha256(y) == str(g["y_sha256/" + key]), key
        y = torch.from_numpy(y).permute(1, 2, 0)[None].contiguous().to(cuda_dev)
        boxes = torch.tensor([f["rect"]], dtype=torch.float32, device=cuda_dev)
        fg = torch.from_numpy(f["fg"][None].astype(np.uint8)).to(cuda_dev) if f["fg"] is not None else None
        out = ops.normal_unwarp(y, boxes, fg, f["H"], f["W"]).cpu().numpy()[0]
        assert np.array_equal(out, g["png/" + key]), (key, int((out != g["png/" + key]).sum()))
    # two frames of one size in one launch: each as on its own
    keys = ["seqA|.|0", "seqA|.|2"]
    fs = [N.prepare_frame(os.path.join(str(tmp_path), "seqA", "imgs", "%s.png" % k[-1])) for k in keys]
    y = torch.stack([torch.from_numpy(R.standin(f["x"])).permute(1, 2, 0) for f in fs]).to(cuda_dev)
    out = ops.normal_unwarp(y.contiguous(), torch.tensor([f["rect"] for f in fs], dtype=torch.float32, device=cuda_dev),
                            torch.from_numpy(np.stack([f["fg"] for f in fs]).astype(np.uint8)).to(cuda_dev), 72, 96)
    for i, k in enumerate(keys):
        assert np.array_equal(out[i].cpu().numpy(), g["png/" + k])


def test_generate_normals_end_to_end(tmp_path, cuda_dev, capsys, monkeypatch):
    dropin()
    from selfreconcode_b200 import normals as N
    from selfreconcode_b200 import synth
    root = synth.write_frame_sequence(str(tmp_path / "seq"), 6, 120, 90, seed=4, normals=False)
    imgs = os.path.join(root, "imgs")
    for i, rect in ((0, [10, 5, 80, 80]), (3, [[-5, -5, 60, 60], [0, 10, 100, 100]])):
        np.savetxt(os.path.join(imgs, "%06d_rect.txt" % i), np.array(rect), fmt="%d")
    twin = R.seeded_net(11, **R.SMALL)
    weights = str(tmp_path / "pifuhd.pt")
    torch.save({"model_state_dict": {"netG.netF." + k: v.float() for k, v in twin.state_dict().items()}}, weights)
    monkeypatch.setattr(N, "MAX_BATCH", 4)              # batches of 4 and 2 here, one of 6 from the command line
    written = N.generate_normals(imgs, weights, device=cuda_dev.index or 0)
    names = sorted(os.listdir(os.path.join(root, "normals")))
    assert names == ["%06d.png" % i for i in range(6)] + ["video.avi"]
    src = [written[os.path.join(root, "normals", "%06d.png" % i)] for i in range(6)]
    assert src[0] == src[3] == "file" and all(src[i] in ("mask", "centre") for i in (1, 2, 4, 5)), src
    assert "mask" in src
    import cv2
    net = N.load_front_net(weights, cuda_dev)
    frames = [N.prepare_frame(os.path.join(imgs, "%06d.png" % i)) for i in range(6)]
    x = torch.from_numpy(np.stack([f["x"] for f in frames]))
    got_n = net(x.to(cuda_dev)).double().cpu()
    ref_n = torch.cat([R.forward64(twin, x[i:i + 1], cuda_dev).cpu() for i in range(6)])
    err = float((got_n - ref_n).abs().max())
    tol = 127.5 * err * 1.01 + 1e-4
    n_near = 0
    for f, rn in zip(frames, ref_n):
        png = cv2.imread(os.path.join(root, "normals", f["name"] + ".png"))
        v, zero = R.unwarp_quantise(rn.numpy(), f["rect"], f["fg"], f["H"], f["W"])
        want = v.astype(np.uint8)
        diff = np.abs(png.astype(np.int64) - want.astype(np.int64))
        frac = v - np.floor(v)
        near = (np.minimum(frac, 1 - frac) <= tol) & ~zero[..., None]
        n_near += int(near.sum())
        assert (diff[~near] == 0).all() and (diff <= 1).all(), f["name"]
    print("end to end: net max |d| %.3g vs the twin; %d channel values within %.3g of an integer" % (err, n_near, tol))
    # the command line, as generate_normals.py's, in one batch: the same files bit for bit
    first = {f["name"]: cv2.imread(os.path.join(root, "normals", f["name"] + ".png")) for f in frames}
    import shutil
    shutil.rmtree(os.path.join(root, "normals"))
    monkeypatch.setattr(N, "MAX_BATCH", 16)
    N.main(["--imgpath", imgs, "--weights", weights, "--gid", str(cuda_dev.index or 0)])
    for name, a in first.items():
        assert np.array_equal(cv2.imread(os.path.join(root, "normals", name + ".png")), a), name
    # the training loader then keeps the sequence's frames on the device with normals
    from dataset.dataset import getDatasetAndLoader
    from model import getOptNet
    sk = synth.make_skinner(resolution=(9, 13, 5))
    g = torch.Generator().manual_seed(1)
    torch.save({"ws": sk.ws, "bmins": sk.b_min, "bmaxs": sk.b_max, "Js": sk.Js, "parents": sk.parents,
                "init_pose": sk.init_pose, "tmpBodyVs": torch.rand(30, 3, generator=g),
                "tmpBodyFs": torch.randint(0, 30, (40, 3), generator=g)}, os.path.join(root, "initial_skinner_1.pth"))
    dataset, loader = getDatasetAndLoader(root, {"deformer": 128, "render": 16}, 2, True, 0, True, True, False)
    getOptNet(dataset, 2, None, None, [(9, 13, 5), (17, 25, 9)], cuda_dev, synth.reference_config())
    capsys.readouterr()
    ids, outs = next(iter(loader))
    log = capsys.readouterr().out
    assert "[frame store] 6 frames of 120x90 with normals" in log, log
    assert "normal" in outs and outs["normal"].is_cuda and outs["normal"].shape == (2, 120, 90, 3)
    for j, i in enumerate(ids.tolist()):
        png = cv2.imread(os.path.join(root, "normals", "%06d.png" % i))
        want = 2. * png[:, :, ::-1].astype(np.float32) / 255. - 1.
        assert np.array_equal(outs["normal"][j].cpu().numpy(), want)
