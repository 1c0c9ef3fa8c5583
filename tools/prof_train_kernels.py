"""Kernels of the training engine at benchmark-like sizes, for `ncu --set full` captures:
    ncu --set full --clock-control none --import-source on -k regex:tc_wgrad_kernel -c 1 -o prof_wgrad python tools/prof_train_kernels.py
    ncu ... -k regex:tc_sweep_kernel -c 40 ...   (forward 4-row <1,4,0> and reverse 4-row <1,4,1> instances among them)
Runs: the 512x512 weight-gradient GEMM over 393 216 rows; one eikonal forward + backward of the full-size SDF on
16 384 points (4 rows per point = 65 536 rows)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    from selfreconcode_b200 import synth
    ms, fl = bench.wgrad_roofline(dev)
    print("wgrad 512x512 over 393216 rows: %.3f ms, %.1f TFLOP/s fp32-equivalent" % (ms, fl / ms / 1e9))
    sdf = synth.make_sdf().to(dev)
    g = torch.Generator().manual_seed(0)
    d = torch.nn.functional.normalize(torch.randn(16384, 3, generator=g), dim=1)
    pts = (d * (0.6 + 0.02 * torch.randn(16384, 1, generator=g))).to(dev)
    for it in range(3):
        sdf.zero_grad()
        q = pts.clone().requires_grad_(True)
        e0, e1, e2 = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e0.record()
        gf = sdf.forward_train(q, 1.0, want_grad=True, want_feat=False)[1]
        loss = ((gf.norm(2, dim=-1) - 1) ** 2).mean()
        e1.record()
        loss.backward()
        e2.record()
        torch.cuda.synchronize()
        print("eikonal on 16384 points: forward %.2f ms, backward %.2f ms" % (e0.elapsed_time(e1), e1.elapsed_time(e2)))


if __name__ == "__main__":
    main()
