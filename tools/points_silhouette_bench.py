"""Device time of the soft point silhouette (ops.points_silhouette: bin, sorts, forward; then backward) on the synthetic
deformed template, and of one whole OptimNetwork.forward with the term on the built-in point renderer, by CUDA events.
Prints the card, its power limit and the template's vertex count beside the numbers.

    python tools/points_silhouette_bench.py [--reps 10]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CASES = [(3, 512, 0.006), (1, 1080, 0.0041)]      # (frames, image side, radius): coarse and fine levels of config.conf


def _card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        pl = pl.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return "%s, power limit %s" % (name, pl)


def _median_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import helpers as H
    H.dropin()
    import test_gpu_mesh_shade as T
    from selfreconcode_b200 import ops
    from model.raster import screen_vertices
    print(_card())
    for n, side, r in CASES:
        net, data, cams, TmpVs, Tmpfs, fids = T._scene(side, side, n)
        poses, trans, d_cond, _ = data.get_grad_parameters(fids, "cuda")
        with torch.no_grad():
            dv = net.deformer(TmpVs[None].expand(n, -1, 3), [d_cond, [poses, trans]], ratio=H.RATIO)
            pts = screen_vertices(dv, cams).contiguous()
        pts.requires_grad_(True)
        g = torch.randn(n, side, side, 1, device="cuda")
        fwd = lambda: ops.points_silhouette(pts, side, side, r, 50)
        both = lambda: torch.autograd.grad(fwd(), [pts], g)
        tf, tb = _median_ms(fwd, a.reps), _median_ms(both, a.reps)
        print("%d frame(s) %dx%d r=%g K=50, template %d vertices: forward %.3f ms, forward+backward %.3f ms "
              "(median of %d)" % (n, side, side, r, TmpVs.shape[0], tf, tb, a.reps))
    print("OptimNetwork.forward + loss.backward (3 frames 512x512, coarse level r=0.006, built-in point renderer): "
          "%.2f ms (median of %d)"
          % (_forward_ms(a.reps), a.reps))


def _forward_ms(reps):
    import helpers as H
    import utils
    from selfreconcode_b200 import synth
    from test_gpu_mesh_shade import _gts, _scene
    side = 512
    net, data, cams, _, _, fids = _scene(side, side, 3)
    conf = synth.reference_config()
    for lvl in ('loss_coarse', 'loss_medium', 'loss_fine'):
        conf[lvl] = dict(conf[lvl], pc_weight=dict(weight=60., mask_weight=1., laplacian_weight=-10.,
                                                   edge_weight=-10., norm_weight=-0.001,
                                                   def_consistent=dict(weight=0.1, c=0.005)))
    net, _ = utils.set_hierarchical_config(conf, 'coarse', net, torch.utils.data.DataLoader(list(range(3)), 3),
                                           synth.MC_LADDER_65)
    datas = {'img': torch.rand(3, side, side, 3, device="cuda") * 2 - 1, 'mask': _gts(3, side, side, False)['mask']}
    net.forward(datas, 2048, H.RATIO, fids)          # first step: hierarchy switch + remesh

    def step():
        net.forward_time = 1                         # no remesh inside the timed steps
        loss = net.forward(datas, 2048, H.RATIO, fids)
        loss.backward()
    return _median_ms(step, reps)


if __name__ == "__main__":
    main()
