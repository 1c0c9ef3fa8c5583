"""Singular values of 3x3 matrices on the device (csrc/svals3x3.cu) at the edges the def_regu term meets and a few it
should survive, against float64 `torch.linalg.svd` of the same fp32 input.

  * forward: J = I, I + eps E (eps 1e-4, 1e-6: three nearly equal values, where def_regu lives early in training),
    exactly repeated values (scaled rotations, diag(2, 2, 0.5)), det < 0, rank 2 and rank 1, overall scales 1e-8 ..
    1e8.  Bar: |S - S64| <= FLT_EPSILON * s_max per matrix (the fp32 rounding of the result is half of that).
  * backward with the def_regu cotangent g_i = dGM(sum_j log^2 s_j)/ds_i, a symmetric function of S: its gradient
    U diag(g) V^T is defined at repeated values too and is compared in float64.  Rank-deficient matrices take the
    cotangent of the sum of the non-zero values (U_r V_r^T).  A J of scale 1e-21 keeps its gradient: the kernel's cut
    for a dropped term is relative to s_max.  A collapsing J (s_min / s_max = 1e-3, 1e-6, 1e-8, the last below
    FLT_EPSILON) keeps def_regu's large restoring term g_min u_min v_min^T.
  * NaN / inf rows leave every other row untouched; n = 0, 1, 257 and one grid-stride pass (132 SMs x 8 CTAs x 256
    threads) plus 1 000; want_v=False gives the same S."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

F32_EPS = 2.0 ** -23
GRID_PASS = 132 * 8 * 256
C_GM = 0.5          # the def_regu GM scale of the shipped configuration


def _rot(g, n):
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).view(n, 3, 3)


def _cases():
    """name -> (J fp32 [n,3,3], rank)"""
    g = torch.Generator().manual_seed(11)
    n = 64
    eye = torch.eye(3, dtype=torch.float64).expand(n, 3, 3)
    E = torch.randn(n, 3, 3, generator=g, dtype=torch.float64)
    R = _rot(g, n)
    U, V = _rot(g, n), _rot(g, n)
    sv = torch.rand(n, 3, generator=g, dtype=torch.float64) + 0.5
    general = U @ torch.diag_embed(sv) @ V.transpose(1, 2)
    out = {
        "identity": (eye, 3),
        "I+1e-4E": (eye + 1e-4 * E, 3),
        "I+1e-6E": (eye + 1e-6 * E, 3),
        "scaled rotation": (R * (0.5 + torch.rand(n, 1, 1, generator=g, dtype=torch.float64)), 3),
        "diag(2,2,0.5)": (U @ torch.diag_embed(torch.tensor([2., 2., .5], dtype=torch.float64).expand(n, 3))
                          @ V.transpose(1, 2), 3),
        "det<0": (general * torch.tensor([1., 1., -1.], dtype=torch.float64).view(1, 1, 3), 3),
        "rank 2": (U @ torch.diag_embed(sv * torch.tensor([1., 1., 0.], dtype=torch.float64)) @ V.transpose(1, 2), 2),
        "rank 1": (U @ torch.diag_embed(sv * torch.tensor([1., 0., 0.], dtype=torch.float64)) @ V.transpose(1, 2), 1),
    }
    # a collapsing J: s_min on both sides of FLT_EPSILON * s_max, where J v / s stops carrying u_min
    for r in (1e-3, 1e-6, 1e-8):
        out["s_min/s_max %.0e" % r] = (U @ torch.diag_embed(torch.tensor([1., .7, r], dtype=torch.float64).expand(n, 3))
                                       @ V.transpose(1, 2), 3)
    for e in (-21, -8, -4, 0, 4, 8):
        out["scale 1e%d" % e] = (general * 10.0 ** e, 3)
    return {k: (v.float().contiguous(), r) for k, (v, r) in out.items()}


def _def_regu_cotangent(S):
    """d/dS of GM(sum log^2 S, c) (utils.GMRobustError with square=True), float64."""
    x = (torch.log(S) ** 2).sum(1, keepdim=True)
    k = 1.0 / (C_GM * C_GM)
    dgm = 2.0 * k * 4.0 / (x * k + 4.0) ** 2
    return dgm * 2.0 * torch.log(S) / S


def test_svals_edges_forward_backward(cuda_dev):
    from selfreconcode_b200 import ops
    worst_s, worst_g = 0.0, 0.0
    for name, (J, rank) in _cases().items():
        U64, S64, Vh64 = torch.linalg.svd(J.double())
        S, V = ops.svals3x3(J.to(cuda_dev), want_v=True)
        S = S.cpu().double()
        es = float(((S - S64).abs().max(1).values / S64[:, 0]).max())
        assert torch.all(S[:, :-1] >= S[:, 1:]), name
        if rank == 3:
            gS = _def_regu_cotangent(S64)
        else:
            gS = (torch.arange(3).view(1, 3) < rank).double().expand_as(S64).contiguous()
        ref = U64 @ torch.diag_embed(gS) @ Vh64
        gJ = ops.svals3x3_backward(J.to(cuda_dev), S.float().to(cuda_dev), V, gS.float().to(cuda_dev)).cpu().double()
        eg = float(((gJ - ref).flatten(1).norm(dim=1) / gS.norm(dim=1).clamp(min=1e-300)).max())   # J = I: g = 0
        print("svals3x3 %-16s |S-S64|/s_max %.2e  |gJ-U diag(g) V^T|/|g| %.2e" % (name, es, eg))
        worst_s, worst_g = max(worst_s, es), max(worst_g, eg)
        assert es <= F32_EPS, (name, es)
        assert eg <= 5e-7, (name, eg)
    print("svals3x3 edges: max S error %.2e s_max (bar %.2e), max backward error %.2e |g| (bar 5e-7)"
          % (worst_s, F32_EPS, worst_g, ))


@pytest.mark.parametrize("n", [0, 1, 257, GRID_PASS + 1000])
def test_svals_sizes_nonfinite_rows_and_want_v(n, cuda_dev):
    from selfreconcode_b200 import ops
    g = torch.Generator().manual_seed(n + 1)
    J = (torch.eye(3).expand(n, 3, 3) + 0.3 * torch.randn(n, 3, 3, generator=g)).contiguous()
    bad = {}
    if n >= 257:
        J[5, 1, 2] = math.nan
        J[100, 0, 0] = math.inf
        J[256, 2, 1] = -math.inf
        bad = {5, 100, 256}
    S, V = ops.svals3x3(J.to(cuda_dev), want_v=True)
    S2, V2 = ops.svals3x3(J.to(cuda_dev), want_v=False)
    assert S.shape == (n, 3) and V2 is None
    assert torch.equal(S, S2)
    ok = torch.ones(n, dtype=torch.bool)
    ok[list(bad)] = False
    S = S.cpu().double()
    if n:
        S64 = torch.linalg.svdvals(J[ok].double())
        err = float(((S[ok] - S64).abs().max(1).values / S64[:, 0]).max())
        print("svals3x3 n=%d: max |S-S64|/s_max %.2e over the finite rows" % (n, err))
        assert err <= F32_EPS
        assert torch.isfinite(S[ok]).all()
        gS = torch.randn(n, 3, generator=g)
        gJ = ops.svals3x3_backward(J.to(cuda_dev), S.float().to(cuda_dev), V, gS.to(cuda_dev)).cpu()
        assert torch.isfinite(gJ[ok]).all()
