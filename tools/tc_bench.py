"""Throughput of one wgmma split-BF16 layer (512x512) vs the FFMA engine's per-layer rate."""
import json, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from selfreconcode_b200 import ops
from selfreconcode_b200._lib import SR_ACT_SOFTPLUS100
dev = torch.device("cuda:0")
out = {}
import os as _os
for M in ((262144,) if _os.environ.get('TC_BENCH_QUICK') else (8192, 50333, 65536, 262144)):
    x = torch.randn(M, 512, device=dev); w = torch.randn(512, 512, device=dev) / 22.6; b = torch.zeros(512, device=dev)
    A = ops.tc_pack_rows(x); W = ops.tc_pack_weights(w)
    ts = []
    for i in range(6):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.tc_linear(A, W, b, M, 512, 512, 512, SR_ACT_SOFTPLUS100, K_next=512)
        e.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(e))
    t = float(np.median(ts[1:]))
    out["M%d_ms" % M] = t
    out["M%d_fp32equiv_TFLOPs" % M] = 2.0 * M * 512 * 512 / t / 1e9
    out["M%d_bf16_TFLOPs" % M] = 6 * 2.0 * M * 512 * 512 / t / 1e9
print(json.dumps(out))
