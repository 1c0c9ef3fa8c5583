"""Time of the normal-map step (selfreconcode_b200/normals.py) on the device, PIFuHD's front-normal net shape
(GlobalGenerator 3 -> 3, ngf 64, 4 downsamplings, 9 blocks, 512 x 512) with seeded weights (torch's default init):

  layers : ms per frame at B = 1 and B = 16, CUDA events after warm-up, broken down by layer kind -- first (7x7,
           3 -> 64), down (4 x 3x3 s2), res (18 x 3x3, 1024 channels), up (4 x ConvTranspose in gather form), last
           (7x7, 64 -> 3, tanh) -- each the im2col pack + tensor-core GEMM, and apart from them the instance norms
           and the unwarp onto a 1080 x 1080 frame;
  cuDNN  : the same weights through the torch twin (tests/normal_net_ref.py) in float32 with TF32 off and on;
  end to end: frames/s of generate_normals over a seeded 64-frame 1080 x 1080 sequence (PNG decode / encode included;
           frames 0, 2, 4, ... carry a _rect.txt, the others take their box from the mask).
Prints the card and its power limit, then one JSON line.

    python tools/normals_bench.py [--out DIR] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        pl = pl.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return "%s, power limit %s" % (name, pl)


def _timed_forward(net, x, ev):
    """FrontNormalNet.forward_cl with an event pair around every launch group: ev[kind] += [(start, end), ...]."""
    from selfreconcode_b200 import _lib, ops

    def rec(kind, fn, *a, **k):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        r = fn(*a, **k)
        e.record()
        ev.setdefault(kind, []).append((s, e))
        return r

    def conv_in(kind, h, conv, relu=True, residual=None):
        y = rec(kind, ops.conv2d, h, conv, net.workspace)
        mean, rstd = rec("instance norm", ops.instance_norm_stats, y)
        return rec("instance norm", ops.instance_norm_apply, y, mean, rstd, residual=residual, relu=relu, out=y)
    h = conv_in("first", x, net.first)
    for c in net.down:
        h = conv_in("down", h, c)
    for c1, c2 in net.blocks:
        h = conv_in("res", conv_in("res", h, c1), c2, relu=False, residual=h)
    for c in net.up:
        h = conv_in("up", h, c)
    return rec("last", ops.conv2d, h, net.last, net.workspace, act=_lib.SR_ACT_TANH)


def bench_layers(net, B, reps):
    from selfreconcode_b200 import ops
    g = torch.Generator().manual_seed(B)
    x = (torch.rand(B, 512, 512, 3, generator=g) * 2 - 1).cuda()
    boxes = torch.tensor([[100, 80, 880, 880]] * B, dtype=torch.float32, device="cuda")
    fg = torch.ones((B, 1080, 1080), dtype=torch.uint8, device="cuda")
    for _ in range(2):
        net.forward_cl(x)
    torch.cuda.synchronize()
    tot = {}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    whole = []
    for _ in range(reps):
        ev = {}
        s.record()
        out = _timed_forward(net, x, ev)
        s2, e2 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s2.record()
        ops.normal_unwarp(out, boxes, fg, 1080, 1080)
        e2.record()
        ev.setdefault("unwarp", []).append((s2, e2))
        e.record()
        torch.cuda.synchronize()
        whole.append(s.elapsed_time(e))
        for k, v in ev.items():
            tot[k] = tot.get(k, 0.0) + sum(a.elapsed_time(b) for a, b in v)
    res = {k: v / reps / B for k, v in tot.items()}
    res["total"] = float(np.median(whole)) / B
    return res


def bench_cudnn(twin, B, reps, tf32):
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    x = torch.rand(B, 3, 512, 512, device="cuda") * 2 - 1
    with torch.no_grad():
        for _ in range(2):
            twin(x)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            twin(x)
        e.record()
        torch.cuda.synchronize()
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = False
    return s.elapsed_time(e) / reps / B


def bench_end_to_end(weights, F=64, H=1080, W=1080):
    from selfreconcode_b200 import enable_dropin, normals, synth
    enable_dropin()
    with tempfile.TemporaryDirectory() as d:
        root = synth.write_frame_sequence(os.path.join(d, "seq"), F, H, W, seed=3, normals=False)
        for i in range(0, F, 2):
            np.savetxt(os.path.join(root, "imgs", "%06d_rect.txt" % i), np.array([[60, 20, 960, 960]]), fmt="%d")
        normals.generate_normals(os.path.join(root, "imgs"), weights, 0)   # warm-up run
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        written = normals.generate_normals(os.path.join(root, "imgs"), weights, 0)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        assert len(written) == F
    return F / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "normals_bench needs a GPU"
    card = _card()
    print("card:", card, flush=True)
    import normal_net_ref as R
    from selfreconcode_b200 import normals
    twin = R.seeded_net(0, **normals.PIFUHD_ARCH).float()
    sd = {k: v.clone() for k, v in twin.state_dict().items()}
    net = normals.load_front_net(sd, "cuda:0")
    res = {"card": card, "layers_ms_per_frame": {}}
    for B in (1, 16):
        r = bench_layers(net, B, args.reps)
        res["layers_ms_per_frame"]["B%d" % B] = {k: round(v, 3) for k, v in r.items()}
        print("B=%d:" % B, res["layers_ms_per_frame"]["B%d" % B], flush=True)
    twin = twin.cuda().eval()
    res["cudnn_fp32_ms_per_frame_B16"] = round(bench_cudnn(twin, 16, args.reps, False), 3)
    res["cudnn_tf32_ms_per_frame_B16"] = round(bench_cudnn(twin, 16, args.reps, True), 3)
    print("cuDNN fp32 %.3f ms/frame, tf32 %.3f ms/frame" % (res["cudnn_fp32_ms_per_frame_B16"],
                                                           res["cudnn_tf32_ms_per_frame_B16"]), flush=True)
    del twin, net
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as d:
        w = os.path.join(d, "pifuhd.pt")
        torch.save({"model_state_dict": {"netG.netF." + k: v for k, v in sd.items()}}, w)
        res["end_to_end_frames_per_s_64x1080x1080"] = round(bench_end_to_end(w), 2)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "normals_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
