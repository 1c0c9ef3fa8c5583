"""A/B timing on the same GPU: the reference's own CUDA extensions (built from /root/reference sources
into oracle/_ref/ by oracle/build.py) vs this library's kernels for the same calls ("kernel to beat",
SURVEY.md 8d).  Measurement tooling, not product code: like tests/ it loads the checker artefacts under oracle/_ref/;
nothing in selfreconcode_b200/ depends on it.  CUDA events, median of 10 after 3 warm-ups, whole call as the reference's user makes it."""
import json, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import selfreconcode_b200
selfreconcode_b200.enable_dropin()
from oracle import build as obuild
import FastMinv, MCGpu, interp2x_boundary3d, GridSamplerMine
dev = torch.device("cuda:0")


def timeit(fn, n=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


out = {}
g = torch.Generator(device=dev).manual_seed(0)
# ---- marching cubes 257^3 on a lumpy sphere
ax = torch.linspace(-1, 1, 257, device=dev)
xx, yy, zz = torch.meshgrid(ax, ax, ax, indexing="ij")
grid = (torch.sqrt(xx * xx + yy * yy + zz * zz) - 0.6 + 0.05 * torch.sin(7 * xx) * torch.cos(5 * yy)).contiguous()
ref = obuild.load_ref("MCGpu")
args = (grid, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.0)
out["mc257_ours_ms"] = timeit(lambda: MCGpu.mc_gpu(*args))
if ref is not None:
    out["mc257_ref_ms"] = timeit(lambda: ref.mc_gpu(*args))
    v, f = MCGpu.mc_gpu(*args); vr, fr = ref.mc_gpu(*args)
    out["mc257_faces"] = [int(f.shape[0]), int(fr.shape[0])]
# ---- 3x3 inverse, 1M matrices
ms = torch.randn(1 << 20, 3, 3, device=dev, generator=g)
ref = obuild.load_ref("FastMinv")
out["minv1M_ours_ms"] = timeit(lambda: FastMinv.Fast3x3Minv(ms))
if ref is not None:
    out["minv1M_ref_ms"] = timeit(lambda: ref.Fast3x3Minv(ms))
# ---- interp2x + boundary 129^3 -> 257^3
occ = grid[::2, ::2, ::2].contiguous().view(1, 1, 129, 129, 129)
ref = obuild.load_ref("interp2x_boundary3d")
out["interp2x_129_ours_ms"] = timeit(lambda: interp2x_boundary3d.forward(occ, 0.0))
if ref is not None:
    out["interp2x_129_ref_ms"] = timeit(lambda: ref.forward(occ, 0.0))
# ---- grid sampler: 24-channel skin-weight volume, 1M points (the LBS lookup)
ws = torch.rand(1, 24, 65, 225, 129, device=dev, generator=g)
pts = (torch.rand(1, 1, 1, 1 << 20, 3, device=dev, generator=g) * 2 - 1)
ref = obuild.load_ref("GridSamplerMine")
out["gridsample_1M_ours_ms"] = timeit(lambda: GridSamplerMine.forward(ws, pts, 0, 1))
if ref is not None:
    out["gridsample_1M_ref_ms"] = timeit(lambda: ref.forward(ws, pts, 0, 1))
    go = torch.randn(1, 24, 1, 1, 1 << 20, device=dev, generator=g)
    out["gridsample_bwd_1M_ours_ms"] = timeit(lambda: GridSamplerMine.backward(ws, pts, go, 0, 1))
    out["gridsample_bwd_1M_ref_ms"] = timeit(lambda: ref.backward(ws, pts, go, 0, 1))
print(json.dumps(out))
