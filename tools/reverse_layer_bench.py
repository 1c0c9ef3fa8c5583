"""Times the tensor-core layer launches of a reverse sweep against the forward launch of the same GEMM (CUDA events).

  python tools/reverse_layer_bench.py [--lib PATH] [--M 50333] [--launches 48] [--windows 5]

At M rows (default: the benchmark frame's 50 333 rays), K = 512:
  * fwd_512   : the 512x512 softplus forward launch (bench.layer_roofline's kernel), the control;
  * rev_512   : the 512x512 reverse launch of a sweep (act' multiply: the previous layer's activation tiles as
                `mul_tiles`, softplus), the same GEMM as fwd_512 plus that operand;
  * rev_N39   : the N = 39 input-gradient launch that ends the SDF's reverse sweep (narrow column tile).
Each launch rotates over 4 operand sets (4 x (in + out) > 50 MB of L2), as the layers of a sweep find their inputs in
HBM.  Every figure is the median over `--windows` windows of `--launches` launches.  gap_ms = rev_512 - fwd_512 is what
the reverse epilogue's extra operand costs.  --lib times another build of the library (SELFRECON_B200_LIB), so that
two builds can be alternated in one session.  Prints one JSON line; the card name and power limit are part of it."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


def _gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       timeout=10).decode().strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="library to time (default: the in-tree build)")
    ap.add_argument("--M", type=int, default=50333)
    ap.add_argument("--launches", type=int, default=48)
    ap.add_argument("--windows", type=int, default=5)
    args = ap.parse_args()
    if args.lib:
        os.environ["SELFRECON_B200_LIB"] = os.path.abspath(args.lib)
    sys.path.insert(0, os.path.abspath(ROOT))
    import torch
    from selfreconcode_b200 import _lib, ops
    from selfreconcode_b200._lib import SR_ACT_NONE, SR_ACT_SOFTPLUS100
    assert torch.cuda.is_available(), "reverse_layer_bench needs a GPU"
    lib = _lib.load()
    dev = torch.device("cuda:0")
    M, K = args.M, 512
    g = torch.Generator(device=dev).manual_seed(5)
    vp = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    W = ops.tc_pack_weights(torch.randn(512, K, device=dev, generator=g) / 22.6)
    Wt = ops.tc_pack_weights(torch.randn(512, K, device=dev, generator=g) / 22.6)   # a reverse launch's W^T
    W39 = ops.tc_pack_weights(torch.randn(39, K, device=dev, generator=g) / 22.6)
    bias = torch.zeros(512, device=dev)
    # layer inputs / sweep deltas, the previous layer's (positive, softplus-like) activations, next-layer tiles
    ins = [ops.tc_pack_rows(torch.randn(M, K, device=dev, generator=g)) for _ in range(4)]
    acts = [ops.tc_pack_rows(torch.rand(M, K, device=dev, generator=g) * 0.05) for _ in range(4)]
    outs = [torch.empty_like(ins[0]) for _ in range(4)]
    out39 = [torch.empty(M, 64, device=dev) for _ in range(4)]

    def fwd(i):
        return lib.sr_tc_linear(vp(ins[i]), vp(W), vp(bias), M, 512, K, 512, SR_ACT_SOFTPLUS100, 1, vp(outs[i]), 512,
                                1.0, None, 0, 0, None, 0, 0, 512, None, None, 0, 0, 1.0, None, st)

    def rev(i):
        return lib.sr_tc_linear(vp(ins[i]), vp(Wt), vp(bias), M, 512, K, 512, SR_ACT_NONE, 1, vp(outs[i]), 512,
                                1.0, None, 0, 0, None, 0, 0, 512, None, vp(acts[i]), 512, SR_ACT_SOFTPLUS100, 1.0,
                                None, st)

    def rev39(i):
        return lib.sr_tc_linear(vp(ins[i]), vp(W39), vp(bias), M, 39, K, 39, SR_ACT_NONE, 1, None, 0, 1.0, None, 0, 0,
                                vp(out39[i]), 64, 0, 39, None, None, 0, 0, 1.0, None, st)

    def timed(fn):
        for i in range(8):
            assert fn(i & 3) == 0
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.windows):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.launches):
                fn(i & 3)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / args.launches)
        return statistics.median(ms), min(ms), max(ms)

    res = {"gpu": _gpu_info(), "lib": _lib.LIB_PATH, "M": M}
    for name, fn in (("fwd_512", fwd), ("rev_512", rev), ("rev_N39", rev39)):
        med, lo, hi = timed(fn)
        res["ms_" + name] = round(med, 5)
        res["range_" + name] = [round(lo, 5), round(hi, 5)]
    res["gap_ms"] = round(res["ms_rev_512"] - res["ms_fwd_512"], 5)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
