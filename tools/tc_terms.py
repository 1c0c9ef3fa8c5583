"""Accuracy / speed of the split-BF16 layer GEMM against fp32 / fp64 references.  Compare the 2-plane (3 terms,
default) and 3-plane (6 terms) builds: build.build_variant("p3", ["SR_TC_PLANES=3"]), then run this script once per
library with SELFRECON_B200_LIB pointing at it."""
import json, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from selfreconcode_b200 import ops, synth
from selfreconcode_b200._lib import SR_ACT_NONE
dev = torch.device("cuda:0")
out = {}
torch.manual_seed(0)
M = 65536
x = torch.randn(M, 512, device=dev); w = torch.randn(512, 512, device=dev) / 22.6; b = torch.zeros(512, device=dev)
A = ops.tc_pack_rows(x); W = ops.tc_pack_weights(w)
y = ops.tc_linear(A, W, b, M, 512, 512, 512, SR_ACT_NONE, want_out=True)[1]
ref = (x[:4096].double() @ w.double().t())
e = (y[:4096].double() - ref)
out["layer_max_rel"] = float(e.abs().max() / ref.abs().max())
out["layer_mean_signed_rel"] = float((e / ref.abs().clamp(min=1e-3)).mean())
y32 = x[:4096] @ w.t()
out["torch_fp32_max_rel"] = float((y32.double() - ref).abs().max() / ref.abs().max())
# full 8x512 SDF: tc engine vs fp64 torch
sdf = synth.make_sdf().to(dev)
g = torch.Generator().manual_seed(5)
pts = ((torch.rand(32768, 3, generator=g) - 0.5) * 1.6).to(dev)
net = sdf.fused_sdf_only(); net.set_pe_weights([1.0] * 6)
s_tc = ops.tc_mlp_forward(net, pts, ch=1, n_out=1).view(-1)
s_ff = ops.sdf_forward(net, pts, False, 0)[0].view(-1)
sd = sdf.double()
with torch.no_grad():
    s64 = sd._forward_autograd(pts.double(), 1.0).view(-1)
out["sdf_tc_vs_fp64_maxabs"] = float((s_tc.double() - s64).abs().max())
out["sdf_ffma_vs_fp64_maxabs"] = float((s_ff.double() - s64).abs().max())
out["sdf_tc_vs_fp64_mean_signed"] = float((s_tc.double() - s64).mean())
out["sdf_scale"] = float(s64.abs().max())
for Mb in (262144,):
    x = torch.randn(Mb, 512, device=dev); A = ops.tc_pack_rows(x)
    ts = []
    for i in range(6):
        a, e2 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); ops.tc_linear(A, W, b, Mb, 512, 512, 512, 1, K_next=512); e2.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(e2))
    out["M%d_ms" % Mb] = float(np.median(ts[1:]))
print(json.dumps(out))
