"""Runs the reference's own CUDA extensions (oracle/_ref/, built by oracle.build.build_ref) on the inputs of the
reference-kernel tests in tests/test_gpu_parity.py and stores their outputs as tests/golden/ref_kernels.npz, so the
tests compare with the reference kernels without needing them.  Needs a GPU:

  python oracle/make_golden_ref_kernels.py [OUT.npz]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main(out):
    from oracle import build
    import test_gpu_parity as T
    dev = torch.device("cuda:0")
    res = {}
    r = build.load_ref("FastMinv")
    ms, gr = [t[:T.MINV_REF_N].to(dev) for t in T._minv_inputs()]
    inv, mask = r.Fast3x3Minv(ms)
    res["minv_inv"], res["minv_mask"] = inv.cpu().numpy(), mask.cpu().numpy()
    res["minv_bwd"] = r.Fast3x3Minv_backward(gr, inv).cpu().numpy()
    r = build.load_ref("MCGpu")
    for n, aniso in T.MC_REF_CASES:
        v, f = r.mc_gpu(T._test_grid(n, 100 + n, aniso).to(dev), *T.MC_REF_ARGS)
        cv, cf = T._canon(v.cpu().numpy(), f.cpu().numpy())
        res["mc%d_verts" % n], res["mc%d_faces" % n] = cv.astype(np.float32), cf.astype(np.int16)
    r = build.load_ref("interp2x_boundary3d")
    x, y = [t.to(dev) for t in T._interp_inputs()]
    o, b = r.forward(x, 0.0)
    res["interp_out"], res["interp_bnd"], res["interp_bwd"] = o.cpu().numpy(), b.cpu().numpy(), r.backward(y).cpu().numpy()
    r = build.load_ref("GridSamplerMine")
    inp, grid, go, ggi, ggg = [t.to(dev) for t in T._grid_sampler_inputs()]
    res["gs_fwd"] = r.forward(inp, grid, 0, 1).cpu().numpy()
    gi, gg = r.backward(inp, grid, go, 0, 1)
    res["gs_bwd_input"], res["gs_bwd_grid"] = gi.cpu().numpy(), gg.cpu().numpy()
    for i, t in enumerate(r.dbackward(ggi, ggg, inp, grid, go, 0, 1)):
        res["gs_dbwd%d" % i] = t.cpu().numpy()
    assert all(len(v) < 32768 for k, v in res.items() if k.endswith("_verts"))   # faces stored as int16
    np.savez_compressed(out, **res)
    print(out, os.path.getsize(out), {k: v.shape for k, v in res.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_kernels.npz"))
