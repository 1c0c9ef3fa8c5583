"""Device time of the template mesh regularisers (ops.mesh_reg_topology; ops.mesh_regularizers forward + backward)
against a torch fp32 restatement of the same three terms on the same GPU, by CUDA events, on synthetic-SDF templates
from two marching-cubes ladders: MC_LADDER_257 and the reference's coarse ladder (train.py, final level 225x321x129).
Both are checked against the same torch terms evaluated in fp64 (the device must agree to elem_err 1e-5 in its
gradient; the fp32 torch error is printed beside it).  Prints the card, its power limit and the mesh sizes beside the
numbers.

    python tools/mesh_reg_bench.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

REF_COARSE = [(15, 21, 9), (29, 41, 17), (57, 81, 33), (113, 161, 65), (225, 321, 129)]
WEIGHTS = (2.0, 30.0, 0.5)      # any positive weights: both sides take the same weighted sum


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
    for _ in range(3):
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


def torch_terms(v, topo):
    """The three terms in torch fp32 ops on the device topology's edges and pairs (scatter-adds: atomics)."""
    V, E, P = topo.V, topo.E, topo.P
    a, b = topo.edges[:, 0], topo.edges[:, 1]
    src, dst = torch.cat([a, b]), torch.cat([b, a])
    deg = torch.zeros(V, dtype=v.dtype, device=v.device).index_add_(0, src, torch.ones_like(src, dtype=v.dtype))
    inv = torch.where(deg > 0, 1.0 / deg.clamp(min=1.0), deg)
    lv = torch.zeros_like(v).index_add_(0, src, v[dst] * inv[src, None]) - v
    lap = lv.norm(dim=1).sum() / V
    edge = ((v[a] - v[b]).norm(dim=1) ** 2).sum() / E
    q = topo.pairs
    va = v[q[:, 0]]
    e1 = v[q[:, 1]] - va
    ni, nj = torch.linalg.cross(e1, v[q[:, 2]] - va, dim=1), torch.linalg.cross(e1, v[q[:, 3]] - va, dim=1)
    cos = (ni * -nj).sum(1) / ((ni * ni).sum(1) * (nj * nj).sum(1)).clamp_min(1e-16).sqrt()
    nc = (1 - cos).sum() / P
    return torch.stack([lap, edge, nc])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import helpers as H
    from selfreconcode_b200 import ops, synth
    from test_gpu_mesh_reg import template
    print(_card())
    w = torch.tensor(WEIGHTS, device="cuda")
    disagree = []
    for label, ladder in (("MC_LADDER_257", synth.MC_LADDER_257), ("reference coarse ladder", REF_COARSE)):
        v, f = template(ladder)
        V = v.shape[0]
        vs = v.clone().requires_grad_(True)
        topo = ops.mesh_reg_topology(f, V)

        def dev():
            return torch.autograd.grad((ops.mesh_regularizers(vs, topo) * w).sum(), [vs])[0]

        def ref():
            return torch.autograd.grad((torch_terms(vs, topo) * w).sum(), [vs])[0]

        t_topo = _median_ms(lambda: ops.mesh_reg_topology(f, V), a.reps)
        t_dev, t_ref = _median_ms(dev, a.reps), _median_ms(ref, a.reps)
        t_dev2 = _median_ms(dev, a.reps)         # alternated: the spread of the device figure
        v64 = vs.detach().double().requires_grad_(True)
        r64 = torch_terms(v64, topo)
        g64, = torch.autograd.grad((r64 * w.double()).sum(), [v64])
        with torch.no_grad():
            r_dev, r_ref = ops.mesh_regularizers(vs, topo), torch_terms(vs, topo)
        rel = lambda r: ((r.double() - r64.detach()).abs() / r64.detach().abs()).max().item()
        g64 = g64.cpu().numpy()
        gerr_dev, gerr_ref = H.elem_err(dev().cpu().numpy(), g64), H.elem_err(ref().cpu().numpy(), g64)
        print("%s %s: V=%d F=%d E=%d P=%d; topology %.3f ms; forward + backward: device %.3f / %.3f ms, torch fp32 "
              "%.3f ms (median of %d); against fp64: values rel %.1e (device) / %.1e (torch fp32), gradient elem_err "
              "%.1e (device) / %.1e (torch fp32)" % (label, ladder[-1], V, topo.F, topo.E, topo.P, t_topo, t_dev, t_dev2,
                                                      t_ref, a.reps, rel(r_dev), rel(r_ref), gerr_dev, gerr_ref))
        if not (rel(r_dev) < 1e-6 and gerr_dev < 1e-5):
            disagree.append(label)
    assert not disagree, "device terms disagree with the fp64 evaluation on %s" % disagree


if __name__ == "__main__":
    main()
