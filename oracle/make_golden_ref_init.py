"""TEST INFRASTRUCTURE -- writes tests/golden/reference_init.npz from the UNMODIFIED reference (imported on CPU through
oracle/ref_shim.py; needs the reference tree, no GPU):

    python oracle/make_golden_ref_init.py [OUT.npz]

  mc_tri_table             a2iTriangleConnectionTable of MCGpu/CudaKernels.cu (tests/test_oracle_c.py)
  sdf/<key>|..., translator/<key>|...
                           getTmpSdf("cpu", 6, bias=0.78) under torch seed 0 and MLPTranslator(128, 6) under seed 1
                           (tests/test_dropin_cpu.py): per state_dict entry the shape, float64 sum and sum of |x|, and
                           64 values at indices drawn from numpy's default_rng(0) in sorted-key order.
"""
import os
import re
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)


def main(out):
    import ref_shim
    src = open(os.path.join(ref_shim.REF_ROOT, "MCGpu", "CudaKernels.cu")).read()
    i = src.index("a2iTriangleConnectionTable[256][16]")
    body = src[src.index("{", i) + 1:src.index("};", i)]
    tab = np.array([[int(x) for x in r.split(",")] for r in re.findall(r"\{([^{}]*)\}", body)], dtype=np.int32)
    ref = ref_shim.load_reference()
    res = {"mc_tri_table": tab}
    rng = np.random.default_rng(0)

    def summarize(prefix, sd):
        for k, v in sorted(sd.items()):
            a = v.detach().double().numpy().reshape(-1)
            idx = np.sort(rng.choice(a.size, size=min(a.size, 64), replace=False))
            res[prefix + k + "|shape"] = np.array(v.shape, dtype=np.int64)
            res[prefix + k + "|idx"] = idx.astype(np.int64)
            res[prefix + k + "|val"] = a[idx].astype(np.float32)
            res[prefix + k + "|sum"] = np.array([a.sum(), np.abs(a).sum()])

    torch.manual_seed(0)
    summarize("sdf/", ref.network.getTmpSdf("cpu", 6, bias=0.78).state_dict())
    torch.manual_seed(1)
    summarize("translator/", ref.Deformer.MLPTranslator(128, 6).state_dict())
    np.savez_compressed(out, **res)
    print(out, os.path.getsize(out), len(res))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "reference_init.npz"))
