"""Times the narrow tensor-core layer launches and the shading call of the ray part (CUDA events, one GPU).

  python tools/narrow_bench.py [--tree DIR] [--M 50333] [--iters 200]

  * N = 1 forward launch (the value-only SDF's last layer, K = 512) and N = 39 reverse launch (the first layer's
    input gradient of the SDF's reverse sweep, K = 512) at M rows -- the shapes of one trace iteration;
  * ops.shade_and_render_tc on M points with the benchmark's networks (synth.make_*).

--tree imports selfreconcode_b200 from another checkout (its library built in place), so that two versions can be
compared in the same process environment.  Prints one JSON line; the card name and power limit are part of it."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys


def _gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       timeout=10).decode().strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    ap.add_argument("--M", type=int, default=50333)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import torch
    from selfreconcode_b200 import _lib, ops, synth
    assert torch.cuda.is_available(), "narrow_bench needs a GPU"
    lib = _lib.load()
    dev = torch.device("cuda:0")
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)   # noqa: E731
    st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)              # noqa: E731
    g = torch.Generator().manual_seed(0)
    M, K = args.M, 512

    def timed(fn, iters):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    A = ops.tc_pack_rows(torch.randn(M, K, generator=g).to(dev))
    res = {"gpu": _gpu_info(), "tree": os.path.abspath(args.tree), "M": M}
    # forward N = 1 (value-only SDF output: out column 0)
    W1 = ops.tc_pack_weights((0.05 * torch.randn(1, K, generator=g)).to(dev))
    b = torch.zeros(256, device=dev)
    out1 = torch.empty(M, 1, device=dev)

    def fwd1():
        assert lib.sr_tc_linear(p(A), p(W1), p(b), M, 1, K, 1, 0, 1, None, 0, 1.0, None, 0, 0, p(out1), 1, 0, 1,
                                None, None, 0, 0, 1.0, None, st()) == 0
    res["ms_fwd_N1_K512"] = timed(fwd1, args.iters)
    # reverse N = 39 (input gradient of the first layer: g_out columns [0, 39))
    W39 = ops.tc_pack_weights((0.05 * torch.randn(39, K, generator=g)).to(dev))
    out39 = torch.empty(M, 64, device=dev)

    def rev39():
        assert lib.sr_tc_linear(p(A), p(W39), p(b), M, 39, K, 39, 0, 1, None, 0, 1.0, None, 0, 0, p(out39), 64, 0,
                                39, None, None, 0, 0, 1.0, None, st()) == 0
    res["ms_rev_N39_K512"] = timed(rev39, args.iters)
    # shading: SDF + translator + renderer at M points
    ratio = {"sdfRatio": 1.0, "deformerRatio": 1.0, "renderRatio": 1.0}
    sdf, tr, rn = synth.make_sdf().to(dev), synth.make_translator().to(dev), synth.make_render().to(dev)
    sk = synth.make_skinner().to(dev)
    poses, trans, dcond = [t.to(dev) for t in synth.make_frame_params(100, 1)]
    full = sdf.fused()
    full.set_pe_weights([1.0] * 6)
    dnet, rnet = tr.fused(ratio), rn.fused(ratio)
    lbs = sk.lbs_state()
    lbs.set_pose(poses, trans)
    pts = (0.8 * (torch.rand(M, 3, generator=g) - 0.5)).to(dev)
    rays = torch.nn.functional.normalize(torch.randn(M, 3, generator=g), dim=1).to(dev)
    bi = torch.zeros(M, dtype=torch.int64, device=dev)
    res["ms_shade_and_render_tc"] = timed(
        lambda: ops.shade_and_render_tc(full, dnet, lbs, rnet, pts, rays, bi, dcond), max(10, args.iters // 10))
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
