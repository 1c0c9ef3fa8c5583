"""Device time of one OptimNetwork.infer call on the synthetic scene, split into raster + shade (the two MeshRenderer
calls: rasteriser, vertex normals, Phong shading) and the ray part (infer_rays: trace + neural colour), by CUDA events.

    python tools/infer_bench.py [--size 512] [--frames 1] [--reps 5]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import helpers as H
    H.dropin()
    import test_gpu_mesh_shade as T
    from model.raster import HardPhongShader, MeshRenderer
    net, data, cams, TmpVs, Tmpfs, fids = T._scene(a.size, a.size, a.frames)
    net.maskRender = MeshRenderer(net.maskRender.rasterizer, HardPhongShader("cuda", cams))
    spans = {"raster+shade": [], "shade only": [], "rays": []}

    def timed(key, fn):
        def run(*args, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*args, **kw)
            e1.record()
            spans[key].append((e0, e1))
            return out
        return run

    class TimedRenderer(MeshRenderer):
        def __call__(self, *args, **kw):
            return timed("raster+shade", super().__call__)(*args, **kw)

    net.maskRender = TimedRenderer(net.maskRender.rasterizer, net.maskRender.shader)
    net.maskRender.shader = timed("shade only", net.maskRender.shader)
    net.infer_rays = timed("rays", net.infer_rays)
    res = []
    for r in range(a.reps + 1):
        for v in spans.values():
            v.clear()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        net.infer(TmpVs, Tmpfs, a.size, a.size, H.RATIO, fids, False, None)
        t1.record()
        torch.cuda.synchronize()
        if r:      # the first call warms up the caches and the vertex / face CSR
            res.append({"infer": t0.elapsed_time(t1),
                        **{k: sum(x.elapsed_time(y) for x, y in v) for k, v in spans.items()}})
    med = {k: sorted(d[k] for d in res)[len(res) // 2] for k in res[0]}
    print("%d frame(s) at %dx%d, template %d vertices / %d faces, median of %d (ms):"
          % (a.frames, a.size, a.size, TmpVs.shape[0], Tmpfs.shape[0], a.reps),
          " ".join("%s %.3f" % kv for kv in med.items()))


if __name__ == "__main__":
    main()
