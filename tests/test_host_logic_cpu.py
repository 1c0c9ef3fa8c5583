"""Host-side logic that needs no GPU: the struct layouts the C ABI reads, the weight-norm helpers and the benchmark's
parity report."""
import ctypes as C

import torch

from selfreconcode_b200 import _lib

def test_struct_layouts_match_header():
    """ctypes mirrors of the structs in include/selfrecon_b200.h: sizes follow from the field lists there
    (7 pointers + 4 ints; 4 pointers + 4 ints)."""
    assert C.sizeof(_lib.WnLayer) == 7 * 8 + 4 * 4
    assert C.sizeof(_lib.TcLayer) == 4 * 8 + 4 * 4
    assert _lib.WnLayer.n.offset == 56


def test_effective_weights_cache_and_fallback():
    """ImplicitNetwork._effective / shared_weights (one weight-norm sub-graph per step) and train_ops.weight_norm_all
    off the GPU: the element-wise torch form, same tensors inside one shared context, no state left behind."""
    from helpers import dropin
    dropin()
    from selfreconcode_b200 import synth, train_ops as T
    sdf = synth.make_sdf()
    L = sdf.num_layers - 1
    lins = [getattr(sdf, "lin%d" % l) for l in range(L)]
    ref = [T.weight_norm_eff(lin.weight_v, lin.weight_g) for lin in lins]
    assert all(torch.equal(a, b) for a, b in zip(T.weight_norm_all(lins), ref))
    assert torch.equal(sdf._effective(3), ref[3])                 # no context: computed on demand
    with sdf.shared_weights():
        got = [sdf._effective(l) for l in range(L)]
        assert all(torch.equal(a, b) for a, b in zip(got, ref))
        assert sdf._effective(2) is got[2]                        # one sub-graph: the same tensor object
    assert sdf._weff is None
    # gradients flow to both parameters through the shared sub-graph
    with sdf.shared_weights():
        (sdf._effective(1).sum() + sdf._effective(1).pow(2).sum()).backward()
    assert lins[1].weight_v.grad is not None and lins[1].weight_g.grad is not None


def test_weight_norm_backward_formula():
    """The closed form csrc/weight_norm.cu implements (gg = <gw, v>/||v||, gv = g/||v|| (gw - v <gw, v>/||v||^2))
    against torch autograd of g v/||v|| in float64."""
    g0 = torch.Generator().manual_seed(2)
    v = torch.randn(7, 13, generator=g0, dtype=torch.float64, requires_grad=True)
    g = torch.randn(7, 1, generator=g0, dtype=torch.float64, requires_grad=True)
    gw = torch.randn(7, 13, generator=g0, dtype=torch.float64)
    (g * v / v.norm(dim=1, keepdim=True) * gw).sum().backward()
    nrm = v.detach().norm(dim=1, keepdim=True)
    s = (gw * v.detach()).sum(1, keepdim=True)
    gg = s / nrm
    gv = g.detach() / nrm * (gw - v.detach() * s / nrm ** 2)
    assert torch.allclose(gg, g.grad, rtol=1e-12, atol=1e-14)
    assert torch.allclose(gv, v.grad, rtol=1e-12, atol=1e-14)


def test_bench_parity_report_counts():
    """bench.parity_report on hand-made inputs: the bar is applied on decision-insensitive rays only, sign differences
    are split by the oracle's own |f| band, the mesh comparison is exact."""
    import os
    import sys
    import numpy as np
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    P = 6
    pts = torch.linspace(0.1, 1.0, P * 3).view(P, 3)
    rgb = torch.linspace(-0.5, 0.5, P * 3).view(P, 3)
    conv = torch.tensor([1, 1, 0, 1, 0, 1], dtype=torch.bool)
    cpu = {"pts": pts.clone(), "rgb": rgb.clone(), "conv": conv.clone(),
           "sensitive": torch.tensor([0, 0, 0, 0, 1, 1], dtype=torch.bool)}
    gpu = {"pts": pts.clone(), "rgb": rgb.clone(), "conv": conv.clone()}
    gpu["pts"][1, 0] += 1e-2          # insensitive ray over tolerance
    gpu["pts"][5, 2] += 1e-2          # sensitive ray over tolerance: reported, not held against the bar
    gpu["conv"][4] = True             # mask flip on a sensitive ray
    gpu["rgb"][0, 1] += 3e-5          # inside 1e-4 |b| + 1e-4 mean|b|
    grid_c = torch.tensor([[-1.0, 2e-6, 0.5], [0.3, -0.2, -4e-6]]).numpy()
    grid_g = torch.tensor([[-1.0, -1e-6, 0.5], [-0.3, -0.2, -4e-6]])      # one flip inside the band, one outside
    calc = torch.ones(2, 3, dtype=torch.bool)
    faces = np.array([[0, 1, 2], [2, 1, 3]], dtype=np.int64)
    verts = np.zeros((4, 3), dtype=np.float32)
    cpu.update(grid=torch.from_numpy(grid_c), calc=calc, faces=faces, verts=verts)
    gpu.update(grid=grid_g, calc=calc.clone(), faces=torch.from_numpy(faces), verts=torch.from_numpy(verts),
               verts_on_oracle_grid=torch.from_numpy(verts), faces_on_oracle_grid=torch.from_numpy(faces[::-1].copy()))
    rep = bench.parity_report(gpu, cpu, band=1e-5)
    assert rep["rays"] == P and rep["rays_decision_sensitive"] == 2
    assert rep["conv_mismatch_all"] == 1 and rep["conv_mismatch_insensitive"] == 0
    assert rep["pts_rays_over_tol_all"] == 2 and rep["pts_rays_over_tol_insensitive"] == 1
    assert rep["rgb_rays_over_tol_insensitive"] == 0
    assert rep["sign_mismatch"] == 2 and rep["sign_mismatch_outside_fp32_band"] == 1
    assert rep["queried_set_mismatch"] == 0 and rep["mc_mesh_identical"] is True
    assert rep["mc_on_oracle_grid_faces_identical"] is False and rep["mc_on_oracle_grid_verts_identical"] is True
