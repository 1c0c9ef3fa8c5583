"""Device time of a new sequence's one-time initialisers at the reference's sizes, each against the torch path it
replaces, in one run:

  * the skin-weight volume (compute_lbswField, model.Deformer variant): 6 890 seeded vertices with 24 skin weights,
    (129, 225, 65) voxels, k = 30, 30 passes.  The blend, the 30 passes and the whole call on the kernels of
    csrc/lbsw_field.cu, and the cdist + top-k + torch smoothing path (chunks of 50 000 rows) they replace; achieved
    candidate distances/s of the blend and bytes/s of the passes.
  * one initializeTmpSDF epoch (5 000 + 1 890 template points) on the tensor-core engine and on the autograd loop
    (SELFRECON_B200_TC_TRAIN=0's path), alternated.

CUDA events, median over --reps runs after one warm-up.  Prints the card and its power limit.

    python tools/init_bench.py [--reps 5] [--epochs 5]
"""
import argparse
import contextlib
import io
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _median_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def torch_field(bmin, bmax, res, verts, ws, k, smooth_times, chunk=50000):
    """The torch path the kernels replace (cdist + top-k per chunk, then the torch smoothing passes)."""
    from utils.LBSWsmpl import voxel_centres
    from model.Deformer import smooth_weights
    W, H, D = res
    pts = voxel_centres(bmin, bmax, res, verts.device)
    out = []
    for part in torch.split(pts, chunk):
        dist, idx = torch.cdist(part, verts).topk(k, dim=-1, largest=False)
        w = 1. / dist.clamp(0.0001, 1.)
        w = w / w.sum(-1, keepdim=True)
        out.append((ws[idx.reshape(-1)] * w.reshape(-1, 1)).reshape(w.shape[0], k, -1).sum(1))
    field = torch.cat(out, dim=0).transpose(0, 1).reshape(1, -1, D, H, W)
    return smooth_weights(field, smooth_times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=5)
    a = ap.parse_args()
    import helpers
    helpers.dropin()
    from points_silhouette_bench import _card
    from selfreconcode_b200 import ops, synth, train_ops
    from model.Deformer import compute_lbswField
    from model.optim import OptimNetwork
    from test_gpu_lbsw import _synth_verts
    print("card: %s" % _card())

    # ---- skin-weight volume
    res, k, passes = (129, 225, 65), 30, 30
    verts, ws, lo, hi = _synth_verts()
    N, V, Cc = res[0] * res[1] * res[2], verts.shape[0], ws.shape[1]
    field = ops.lbsw_field(lo, hi, res, verts, ws, False, k)
    t_blend = _median_ms(lambda: ops.lbsw_field(lo, hi, res, verts, ws, False, k), a.reps)
    t_pass = _median_ms(lambda: ops.lbsw_smooth(field, passes), a.reps)
    t_dev = _median_ms(lambda: compute_lbswField(lo, hi, res, verts, ws, False, k, passes), a.reps)
    t_torch = _median_ms(lambda: torch_field(lo, hi, res, verts, ws, k, passes), a.reps)
    t_torch_blend = _median_ms(lambda: torch_field(lo, hi, res, verts, ws, k, 0), a.reps)
    cand = float(N) * V
    pass_bytes = passes * 2.0 * N * Cc * 4
    diff = float((compute_lbswField(lo, hi, res, verts, ws, False, k, passes) -
                  torch_field(lo, hi, res, verts, ws, k, passes)).abs().max())
    print("compute_lbswField: %d vertices, C=%d, %s voxels, k=%d, %d passes" % (V, Cc, res, k, passes))
    print("  blend      device %8.2f ms  (%.2f T candidate distances/s; torch cdist + top-k blend %.2f ms)" %
          (t_blend, cand / t_blend / 1e9, t_torch_blend))
    print("  %d passes  device %8.2f ms  (%.1f GB moved, %.2f TB/s)" %
          (passes, t_pass, pass_bytes / 1e9, pass_bytes / t_pass / 1e9))
    print("  whole      device %8.2f ms  torch %8.2f ms  (x%.1f); max |device - torch| %.2e" %
          (t_dev, t_torch, t_torch / t_dev, diff))

    # ---- initializeTmpSDF epochs
    g = torch.Generator().manual_seed(4)
    d = torch.randn(6890, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    on = OptimNetwork(synth.make_sdf().cuda(), None, None, None, None)
    on.tmpBodyVs, on.tmpBodyNs = (0.6 * d).cuda(), d.cuda()
    times = {True: [], False: []}
    for r in range(a.epochs + 1):
        for engine in (True, False):
            train_ops.TC_TRAIN_ENABLED = engine
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            with contextlib.redirect_stdout(io.StringIO()):
                on.initializeTmpSDF(1, None, with_normals=True)
            e.record()
            e.synchronize()
            if r > 0:
                times[engine].append(s.elapsed_time(e) / 1e3)
    train_ops.TC_TRAIN_ENABLED = True
    med = {k_: sorted(v)[len(v) // 2] for k_, v in times.items()}
    print("initializeTmpSDF: one epoch (6 890 points, with normals), median of %d alternated" % a.epochs)
    print("  engine %.4f s  autograd loop %.4f s  (x%.1f); 1 200 epochs: %.1f s vs %.1f s" %
          (med[True], med[False], med[False] / med[True], 1200 * med[True], 1200 * med[False]))


if __name__ == "__main__":
    main()
