"""Device time of the texture atlas (selfreconcode_b200.texture) at the reference's settings: a 1680^2 atlas with 50
slots, 120 frames of 1080x1080 of the synthetic deformed template (tests/test_gpu_mesh_shade._scene) under a chart-per-
face-pair UV layout.  CUDA events, median over the frames (add_frame split into the per-vertex / per-face inputs with
the mesh raster, and the per-texel accumulation) and over repeats (finish); host time of write_texture.  Prints the
card, its power limit, the algorithmic bytes and the bandwidth they imply.

    python tools/texture_bench.py [--frames 120] [--reps 5]
"""
import argparse
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _med(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--resolution", type=int, default=1680)
    ap.add_argument("--views", type=int, default=50)
    ap.add_argument("--side", type=int, default=1080)
    a = ap.parse_args()
    import helpers
    helpers.dropin()
    from points_silhouette_bench import _card
    import test_gpu_texture as TT
    from selfreconcode_b200 import ops
    from selfreconcode_b200.texture import TextureBaker, write_texture
    from model.raster import screen_vertices
    print(_card())
    n, side, R, S = a.frames, a.side, a.resolution, a.views
    net, data, cams, TmpVs, Tmpfs = TT.scene(side, n)
    vt, ft = TT.chart_layout(Tmpfs.shape[0])
    baker = TextureBaker(Tmpfs, torch.from_numpy(vt), torch.from_numpy(ft), R, S, 68., 5, "cuda")
    T = baker.texel_index.numel()
    D = torch.cat([TT.deformed(net, data, TmpVs, list(range(b, min(b + 8, n)))) for b in range(0, n, 8)])
    frames = []
    for k in range(n):
        cov = ops.raster_mesh(screen_vertices(D[k:k + 1], cams), Tmpfs, side, side)[0][0, ..., 0] >= 0
        frames.append((torch.from_numpy(TT.smooth_image(k, side)).cuda(), cov))
    t_in, t_acc = [], []
    for k in range(n):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        screen, weight, usable = baker.frame_inputs(D[k], cams, frames[k][1])
        e[1].record()
        baker.accumulate(screen, weight, usable, frames[k][0], k)
        e[2].record()
        torch.cuda.synchronize()
        t_in.append(e[0].elapsed_time(e[1]))
        t_acc.append(e[1].elapsed_time(e[2]))
    out = baker.finish()
    torch.cuda.synchronize()
    t_fin = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        baker.finish()
        e1.record()
        torch.cuda.synchronize()
        t_fin.append(e0.elapsed_time(e1))
    t_w = []
    with tempfile.TemporaryDirectory() as d:
        for _ in range(3):
            t0 = time.perf_counter()
            write_texture(d, out)
            t_w.append(1e3 * (time.perf_counter() - t0))
    count = out["count"].view(-1)[baker.texel_index].long()
    final = out["mask_final"].view(-1)[baker.texel_index]
    acc_bytes = 24 * T                                     # face id, barycentrics, (min alpha, slot) per texel
    fin_bytes = T * (8 + 4 * S + 12 + 1 + 4 + 4) + int(final.sum()) * 4 + 12 * int(count[final].sum())
    fin_ms, acc_ms = _med(t_fin), _med(t_acc)
    print("template %d vertices / %d faces, %d frames of %dx%d, atlas %d^2 with %d covered texels, %d slots "
          "(%.2f GB of slots)" % (TmpVs.shape[0], Tmpfs.shape[0], n, side, side, R, T, S, 20. * S * T / 1e9))
    print("add_frame: inputs + mesh raster %.3f ms, accumulate %.3f ms (median of %d frames); accumulate reads "
          "%.1f MB per frame at least (24 B per covered texel): %.0f GB/s" % (_med(t_in), acc_ms, n, acc_bytes / 1e6,
                                                                           acc_bytes / acc_ms / 1e6))
    print("finish: %.3f ms (median of %d), %.1f MB (alphas of every slot, colours of the filled slots of final "
          "texels, outputs): %.0f GB/s; %d texels final, mean count %.1f"
          % (fin_ms, a.reps, fin_bytes / 1e6, fin_bytes / fin_ms / 1e6, int(final.sum()), float(count.float().mean())))
    print("write_texture (host, cv2): %.1f ms (median of 3)" % _med(t_w))


if __name__ == "__main__":
    main()
