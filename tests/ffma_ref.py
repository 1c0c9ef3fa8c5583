"""Float64 restatement of the fused fp32 field engine (csrc/mlp_core.cuh, csrc/mlp_kernels.cu): the embedded input
of embed_point, the layer stack of run_net (skip connections, all four activations) and the derivatives the kernels
carry forward (grad f, d offset / d p).  It imports nothing from the product: a network is the same list of layer
dicts ops.FusedMLP.fold takes -- v [n, k], g [n] or None, b [n] or None, act (SR_ACT_*), skip (bool).

The model-level pieces (LBS, bone transforms, cardinal rays, the surface finder) are oracle/oracle.py run in float64.

The keyword switches of embed / mlp exist for the negative controls of tests/test_ffma_ref_cpu.py, which show that
the bars there reject a restatement that lacks the term each switch removes."""
import math

import torch
import torch.nn.functional as F

NONE, SP, RELU, TANH = 0, 1, 2, 3
INV_SQRT2 = 1.0 / math.sqrt(2.0)


def annealing_weights(multires, ratio):
    """One weight per band (utils/utils.py:40-46; sin and cos of a band share it)."""
    if ratio is None:
        return [1.0] * multires
    if ratio <= 0:
        return [0.0] * multires
    a = ratio * multires
    return [(1.0 - math.cos(math.pi * min(max(a - b, 0.0), 1.0))) / 2.0 for b in range(multires)]


def embed(x, multires, pe_w, swap_sincos=False):
    """[x, w_0 sin(x), w_0 cos(x), w_1 sin(2x), w_1 cos(2x), ...], each block 3 wide (embed_point's row layout)."""
    x = x.double()
    parts = [x]
    for b in range(multires):
        s, c = torch.sin(x * 2.0 ** b), torch.cos(x * 2.0 ** b)
        if swap_sincos:
            s, c = c, s
        parts += [pe_w[b] * s, pe_w[b] * c]
    return torch.cat(parts, 1)


def effective_weight(L):
    v = L["v"].double()
    if L.get("g") is None:
        return v
    return v * (L["g"].double().view(-1, 1) / v.norm(dim=1, keepdim=True))


def activation(act, z):
    if act == SP:
        return F.softplus(z, beta=100)           # threshold 20 on 100 z, as softplus100()
    if act == RELU:
        return F.relu(z)
    if act == TANH:
        return torch.tanh(z)
    return z


def mlp(layers, inp, d_in, skip_scale=INV_SQRT2, late_stash=False, with_preacts=False):
    """run_net: h_{l+1} = act_l(W_l h_l + b_l); a skip layer's input is cat(h, inp[:, :d_in]) * skip_scale.
    late_stash: the skip appends the first layer's output instead of the embedded input (negative control).
    with_preacts: also returns every layer's pre-activation (ReLU cases exclude units within rounding of 0)."""
    h = inp
    stash = inp[:, :d_in]
    zs = []
    for l, L in enumerate(layers):
        if L.get("skip"):
            h = torch.cat([h, stash], 1) * skip_scale
        z = h @ effective_weight(L).t().to(h.device)
        if L.get("b") is not None:
            z = z + L["b"].double().to(h.device)
        zs.append(z)
        h = activation(L["act"], z)
        if late_stash and l == 0:
            stash = h[:, :d_in]
    return (h, zs) if with_preacts else h


def min_relu_margin(layers, zs):
    """Per row: the smallest |z| over the units of the ReLU layers (inf without any)."""
    m = torch.full((zs[0].shape[0],), math.inf, dtype=torch.float64, device=zs[0].device)
    for L, z in zip(layers, zs):
        if L["act"] == RELU:
            m = torch.minimum(m, z.abs().min(1).values)
    return m


def sdf(layers, pts, multires, pe_w, want_grad=True, **kw):
    """ImplicitNetwork: -> f [P], grad f [P, 3] (autograd), all outputs [P, n_last]."""
    x = pts.double().detach().clone().requires_grad_(want_grad)
    d_in = 3 + 6 * multires
    out = mlp(layers, embed(x, multires, pe_w, kw.pop("swap_sincos", False)), d_in, **kw)
    f = out[:, 0]
    g = torch.autograd.grad(f.sum(), x)[0] if want_grad else None
    return f.detach(), g, out.detach()


def translator_offset(layers, x, multires, pe_w, conds, frame, with_preacts=False):
    """MLPTranslator: offset = mlp(cat(PE(p), conds[frame])) (differentiable in x)."""
    e = embed(x, multires, pe_w)
    h = torch.cat([e, conds.double().to(e.device)[frame]], 1) if conds is not None else e
    return mlp(layers, h, h.shape[1], with_preacts=with_preacts)


def jacobian(fn, pts):
    """fn(x [P, 3]) -> y [P, 3]; returns y and dy/dx [P, 3, 3] (row i = d y_i / d x)."""
    x = pts.double().detach().clone().requires_grad_(True)
    y = fn(x)
    rows = [torch.autograd.grad(y[:, i].sum(), x, retain_graph=i < 2)[0] for i in range(3)]
    return y.detach(), torch.stack(rows, 1)


def render(layers, pts, normals, views, feat, multires, pe_w):
    """RenderingNetwork_view_norm ('idr'): mlp(cat(p, PE(view), n, feature))."""
    parts = [pts.double(), embed(views, multires, pe_w), normals.double()]
    if feat is not None and feat.shape[1]:
        parts.append(feat.double())
    h = torch.cat(parts, 1)
    out, zs = mlp(layers, h, h.shape[1], with_preacts=True)
    return out, min_relu_margin(layers, zs)
