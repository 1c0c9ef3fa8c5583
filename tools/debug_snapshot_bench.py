"""Device time of the `draw` render of OptimNetwork.save_debug on the synthetic scene: trace every covered pixel
(30 iterations), then its colour and camera-frame deformed normal, by CUDA events around the whole render and around
each trace (the rest is the shading).  Two ways, alternated in one session:

    fused  shade_rays(..., deformed_normals=True): the normal comes out of the tensor-core shading pass
           (sr_tc_shade_point_deformed)
    ffma   shade_rays(...) for the colour, then compute_deformed_normals(..., 'test'): grad f and dD/dp evaluated again
           on the fp32 FFMA engine

    python tools/debug_snapshot_bench.py [--size 1080] [--frames 4] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        pl = "unknown"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1080)
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("debug_snapshot_bench: needs a CUDA device")
    import helpers as H
    H.dropin()
    import utils
    import test_gpu_mesh_shade as T
    net, data, cams, TmpVs, Tmpfs, fids = T._scene(a.size, a.size, a.frames)
    N = fids.numel()
    poses, trans, d_cond, _ = data.get_grad_parameters(fids, "cuda")
    defconds = [d_cond.detach(), [poses.detach(), trans.detach()]]
    with torch.no_grad():
        defTmpVs = net.deformer(TmpVs[None].expand(N, -1, 3), defconds, ratio=H.RATIO)
        bi, ri, ci, ps, _ = net._mesh_seed(defTmpVs, TmpVs, Tmpfs)
    cameras, _, _ = net._cameras(N, "cuda")
    R0 = cameras.R[0].detach()
    chunk = 1 << 18
    marks = {}

    def ffma_draw():
        pix = torch.cat([ci.view(-1, 1), ri.view(-1, 1), torch.ones_like(ci.view(-1, 1))], dim=-1)
        rays = cameras.view_rays(pix.float())
        cam_pos = cameras.cam_pos().detach()
        cols, nrms = [], []
        for rays_, ps_, bi_ in zip(torch.split(rays, chunk), torch.split(ps, chunk), torch.split(bi, chunk)):
            ps_, _ = utils.OptimizeSurfacePs(cam_pos, rays_.detach(), ps_.clone(), bi_, net.sdf, H.RATIO, net.deformer,
                                             defconds, dthreshold=1.e-4, athreshold=net.angThred, w1=3.05, w2=1.,
                                             times=30)
            cols.append(utils.shade_rays(net.sdf, net.deformer, net.netRender, ps_, rays_, defconds, bi_, H.RATIO)[2])
            nx, _ = utils.compute_deformed_normals(net.sdf, net.deformer, ps_, defconds, bi_, H.RATIO, 'test')
            nrms.append(utils.camera_normals(nx, R0))
        return torch.cat(cols), torch.cat(nrms)

    def fused_draw():
        return net._draw_rays(bi, ri, ci, ps, cameras, defconds, H.RATIO, chunk=chunk)

    # events around each chunk's trace split the render into trace and shading
    trace = utils.OptimizeSurfacePs

    def traced(*args, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = trace(*args, **kw)
        e1.record()
        marks.setdefault("trace", []).append((e0, e1))
        return out
    utils.OptimizeSurfacePs = traced

    def timed(fn):
        marks.clear()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        with torch.no_grad():
            out = fn()
        e1.record()
        torch.cuda.synchronize()
        total = e0.elapsed_time(e1)
        return total, total - sum(x.elapsed_time(y) for x, y in marks["trace"]), out

    res = {"fused": [], "ffma": []}
    outs = {}
    for r in range(a.reps + 1):
        for k, fn in (("fused", fused_draw), ("ffma", ffma_draw)) if r % 2 == 0 else (("ffma", ffma_draw),
                                                                                        ("fused", fused_draw)):
            t, s, out = timed(fn)
            outs[k] = out
            if r:              # the first round warms up both paths
                res[k].append((t, s))
    utils.OptimizeSurfacePs = trace
    med = lambda v, i: sorted(x[i] for x in v)[len(v) // 2]        # noqa: E731
    name, pl = _card()
    dn = (outs["fused"][1] - outs["ffma"][1]).abs().max().item()
    drgb = (outs["fused"][0] - outs["ffma"][0]).abs().max().item()
    print(json.dumps({"gpu": name, "power_limit,max_sm_clock": pl, "frames": N, "size": a.size,
                      "covered_pixels": int(bi.numel()), "reps": a.reps,
                      "fused_render_ms": med(res["fused"], 0), "ffma_render_ms": med(res["ffma"], 0),
                      "fused_shading_ms": med(res["fused"], 1), "ffma_shading_ms": med(res["ffma"], 1),
                      "all_fused_ms": [round(x[0], 3) for x in res["fused"]],
                      "all_ffma_ms": [round(x[0], 3) for x in res["ffma"]],
                      "max_normal_diff": dn, "max_rgb_diff": drgb}))


if __name__ == "__main__":
    main()
