"""GPU: the training half of the tensor-core engine (selfreconcode_b200/train_ops.py) against plain torch
fp64 autograd of the same computation.

  * sr_tc_wgrad (MN-major wgmma GEMM over the tiled activations) vs delta^T x
  * TcMlpFunction forward / backward with 1 row per point (first order) and 4 rows per point (value + 3 forward
    tangents: the backward contains act'' -- what the reference gets from double backward), incl. the SDF's skip
    connection and narrow first / last layers."""
import numpy as np
import pytest
import torch

from helpers import norm_err

pytestmark = pytest.mark.gpu
SP, RELU, NONE = 1, 2, 0


def _ref_forward(x0, Ws, bs, acts, skips, d_in, ch, relu_masks=None):
    """The forward-mode MLP in differentiable torch ops (any dtype): rows = (point, channel); channel 0 carries the
    value, channels 1..3 tangents that see act'(z_value) and no bias.  `relu_masks[i]` (optional) fixes the ReLU
    on/off pattern of layer i: ReLU's derivative is discontinuous, so two correct evaluations disagree on the few
    units whose pre-activation is within rounding of 0 -- with the product's own pattern the comparison is exact."""
    M = x0.shape[0]
    P = M // ch
    x = x0
    for i, (W, b, act, skip) in enumerate(zip(Ws, bs, acts, skips)):
        if skip:
            x = torch.cat([x[:, :W.shape[1] - d_in], x0[:, :d_in]], dim=1) / np.sqrt(2)
        z = x[:, :W.shape[1]] @ W.t()
        z = z.view(P, ch, -1)
        zv = z[:, 0] + (b if b is not None else 0)
        if act == SP:
            a = torch.nn.functional.softplus(zv, beta=100)
            d = torch.sigmoid(100 * zv)
        elif act == RELU:
            d = (zv > 0).to(zv.dtype) if relu_masks is None else relu_masks[i].to(zv.dtype)
            a = zv * d
        else:
            a, d = zv, torch.ones_like(zv)
        if ch == 1:
            x = a
        else:
            x = torch.cat([a.unsqueeze(1), d.unsqueeze(1) * z[:, 1:]], dim=1).reshape(M, -1)
    return x


def _case(dev, ch, dims, acts, skips, d_in, ld, P, seed):
    g = torch.Generator().manual_seed(seed)
    M = P * ch
    x0 = torch.zeros(M, ld)
    x0[:, :d_in] = torch.randn(M, d_in, generator=g) * 0.5
    Ws, bs = [], []
    k = d_in
    for i, n in enumerate(dims):
        kin = k if not skips[i] else k + d_in
        Ws.append(torch.randn(n, kin, generator=g) / np.sqrt(kin) * (3.0 if acts[i] == SP else 1.4))
        bs.append(torch.randn(n, generator=g) * 0.05)
        k = n
    R = torch.randn(M, dims[-1], generator=g)
    return x0, Ws, bs, R


@pytest.mark.parametrize("swap", [0, 1])
def test_wgrad_matches_fp64(cuda_dev, swap):
    from selfreconcode_b200 import _lib, ops
    from selfreconcode_b200.train_ops import _Workspace
    from selfreconcode_b200.ops import _p, _stream
    lib = _lib.load()
    g = torch.Generator().manual_seed(3)
    res = {}
    for (M, n, k) in ((5000, 512, 512), (777, 257, 64), (20000, 3, 512), (4100, 473, 192)):
        d = torch.randn(M, n, generator=g)
        x = torch.randn(M, k, generator=g)
        Kd, Kx = (n + 127) // 128 * 128, (k + 31) // 32 * 32
        dp = torch.zeros(M, Kd)
        dp[:, :n] = d
        xp = torch.zeros(M, Kx)
        xp[:, :k] = x
        D = ops.tc_pack_rows(dp.to(cuda_dev))
        X = ops.tc_pack_rows(xp.to(cuda_dev))
        part = _Workspace.get(cuda_dev, lib.sr_tc_wgrad_partial_bytes(M, Kd, Kx, None))
        dW = torch.empty(n, k, device=cuda_dev)
        lib.sr_tc_debug_wgrad_desc_swap(swap)
        try:
            rc = lib.sr_tc_wgrad(_p(D), Kd, _p(X), Kx, M, _p(part), _p(dW), n, k, k, _stream())
        finally:
            lib.sr_tc_debug_wgrad_desc_swap(0)
        assert rc == 0
        ref = d.double().t() @ x.double()
        res[(M, n, k)] = norm_err(dW.cpu().numpy(), ref.numpy())
    print("wgrad swap=%d errors:" % swap, res)
    if swap == 0:
        assert max(res.values()) < 2e-5, res
    else:
        assert min(res.values()) > 1e-2, "the swapped descriptor must NOT work (guards the layout reasoning)"


CASES = {
    "relu_ch1": dict(ch=1, dims=[512, 512, 3], acts=[RELU, RELU, NONE], skips=[False] * 3, d_in=167, ld=192, P=3001),
    "relu_ch4": dict(ch=4, dims=[512, 512, 3], acts=[RELU, RELU, NONE], skips=[False] * 3, d_in=167, ld=192, P=700),
    "sdf_ch4": dict(ch=4, dims=[512, 473, 512, 257], acts=[SP, SP, SP, NONE], skips=[False, False, True, False],
                    d_in=39, ld=64, P=650),
    "sdf_ch1": dict(ch=1, dims=[512, 473, 512, 257], acts=[SP, SP, SP, NONE], skips=[False, False, True, False],
                    d_in=39, ld=64, P=2100),
    "small_ch4": dict(ch=4, dims=[64, 64, 1], acts=[SP, SP, NONE], skips=[False] * 3, d_in=39, ld=64, P=300),
    # softplus(beta=100) with |100 z| = O(1): act' and act'' are smooth at the engine's precision, so this case
    # isolates the MACHINERY (4-row reverse epilogue, act'' coupling, skip routing) from the conditioning of beta=100
    "sdf_ch4_gentle": dict(ch=4, dims=[512, 473, 512, 257], acts=[SP, SP, SP, NONE],
                           skips=[False, False, True, False], d_in=39, ld=64, P=650, wscale=0.01),
}
TOL = {"relu_ch1": (1e-4, 3e-4), "relu_ch4": (1e-4, 3e-4), "sdf_ch1": (1e-4, 3e-4), "sdf_ch4_gentle": (1e-4, 3e-4),
       # beta = 100 makes act' = sigmoid(100 z) move by 25 * dz: forward tangents (and what flows back through act'')
       # inherit 25x the engine's ~1e-5 pre-activation error
       "sdf_ch4": (1e-3, 6e-3), "small_ch4": (1e-3, 6e-3)}


@pytest.mark.parametrize("name", list(CASES))
def test_tc_mlp_function_vs_autograd(cuda_dev, name):
    from selfreconcode_b200.train_ops import MlpConfig, tc_mlp
    c = CASES[name]
    from selfreconcode_b200 import train_ops
    x0, Ws, bs, R = _case(cuda_dev, c["ch"], c["dims"], c["acts"], c["skips"], c["d_in"], c["ld"], c["P"], 11)
    if "wscale" in c:
        Ws = [w * c["wscale"] for w in Ws[:-1]] + [Ws[-1]]
        bs = [b * c["wscale"] for b in bs[:-1]] + [bs[-1]]
    # product
    x0g = x0.to(cuda_dev).requires_grad_(True)
    Wg = [w.to(cuda_dev).requires_grad_(True) for w in Ws]
    bg = [b.to(cuda_dev).requires_grad_(True) for b in bs]
    cfg = MlpConfig(c["acts"], c["skips"], c["d_in"], c["ch"])
    train_ops.DEBUG_LAST = {}
    out_g = tc_mlp(x0g, cfg, Wg, bg)
    dbg, train_ops.DEBUG_LAST = train_ops.DEBUG_LAST, None
    masks = None
    if RELU in c["acts"]:      # the product's own ReLU pattern (value rows of the kept activation tiles)
        masks = []
        for i, a in enumerate(dbg["acts"]):
            t = train_ops.unpack_tiles(a, dbg["M"], dbg["widths"][i]).view(-1, c["ch"], dbg["widths"][i])[:, 0]
            masks.append((t > 0).cpu())
        masks.append(None)
    # reference: fp64 autograd
    x0r = x0.double().requires_grad_(True)
    Wr = [w.double().requires_grad_(True) for w in Ws]
    br = [b.double().requires_grad_(True) for b in bs]
    out_r = _ref_forward(x0r, Wr, br, c["acts"], c["skips"], c["d_in"], c["ch"], masks)
    (out_r * R.double()).sum().backward()
    errs = {"out": norm_err(out_g.detach().cpu().numpy(), out_r.detach().numpy())}
    (out_g * R.to(cuda_dev)).sum().backward()
    errs["x0"] = norm_err(x0g.grad.cpu().numpy()[:, :c["d_in"]], x0r.grad.numpy()[:, :c["d_in"]])
    for i in range(len(Ws)):
        errs["W%d" % i] = norm_err(Wg[i].grad.cpu().numpy(), Wr[i].grad.numpy())
        errs["b%d" % i] = norm_err(bg[i].grad.cpu().numpy(), br[i].grad.numpy())
    print(name, {k: "%.1e" % v for k, v in errs.items()})
    assert errs["out"] < TOL[name][0], errs
    assert max(v for k, v in errs.items() if k != "out") < TOL[name][1], errs
    assert (x0g.grad[:, c["d_in"]:] == 0).all()


def test_embed_kernels_match_torch_embedding(cuda_dev):
    """EmbedRowsFunction (embed_kernel / embed_bwd_kernel) vs the differentiable torch restatement: rows, d/dp incl. the
    second derivative that the tangent rows need, d/d(latent code)."""
    from selfreconcode_b200 import train_ops as T
    g = torch.Generator().manual_seed(1)
    for ch, E in ((4, 128), (1, 0), (4, 0), (1, 128)):
        p = (torch.rand(500, 3, generator=g) * 2 - 1).to(cuda_dev)
        ex = torch.randn(500, E, generator=g).to(cuda_dev) if E else None
        pe_w = [1.0, 1.0, 0.7, 0.2, 0.0, 0.0]
        outs = {}
        for mode in (True, False):
            T.EMBED_KERNELS = mode
            pp = p.clone().requires_grad_(True)
            ee = ex.clone().requires_grad_(True) if E else None
            x0 = T.embed_rows(pp, 6, pe_w, ch, extra=ee)
            R = torch.randn(x0.shape, generator=torch.Generator().manual_seed(2)).to(cuda_dev)
            (x0 * R).sum().backward()
            outs[mode] = (x0.detach(), pp.grad, ee.grad if E else None)
        T.EMBED_KERNELS = True
        assert norm_err(outs[True][0].cpu().numpy(), outs[False][0].cpu().numpy()) < 2e-6
        assert norm_err(outs[True][1].cpu().numpy(), outs[False][1].cpu().numpy()) < 1e-5
        if E:
            assert norm_err(outs[True][2].cpu().numpy(), outs[False][2].cpu().numpy()) < 1e-6
