"""Neural SDF (reference: model/network.py:14-118) on the fused CUDA engines.

`ImplicitNetwork` keeps the reference's constructor signature, initialisation, attribute names
and state_dict keys (lin{l}.weight_g / weight_v / bias), and the `rendcond` side effect of
forward().  Execution:
  * no autograd needed (tracing, MC queries, inference): one fused kernel per call
    (csrc/mlp_kernels.cu: sdf_kernel) -- PE, all layers, softplus, optional grad f.
  * autograd needed (training losses with create_graph): the same math as differentiable
    torch ops on the GPU.  (Fused backward kernels are the next step; see DESIGN.md.)
CPU tensors are rejected: there is no CPU path.
"""
import contextlib

import numpy as np
import torch
import torch.nn as nn

from selfreconcode_b200 import ops
from .Embedder import get_embedder
from ._fused import (FoldCache, needs_autograd, ratio_value, require_cuda, SR_ACT_NONE,
                     SR_ACT_SOFTPLUS100)


class ImplicitNetwork(nn.Module):
    def __init__(self, feature_vector_size, d_in, d_out, dims, geometric_init=True, bias=1.0,
                 skip_in=(), weight_norm=True, multires=0):
        super().__init__()
        dims = [d_in] + list(dims) + [d_out + feature_vector_size]
        self.d_out = d_out
        self.embed_fn = None
        self.multires = multires
        if multires > 0:
            self.embed_fn, dims[0] = get_embedder(multires)
        self.num_layers = len(dims)
        self.skip_in = skip_in
        self.weight_norm = weight_norm
        for l in range(self.num_layers - 1):
            out_dim = dims[l + 1] - dims[0] if (l + 1) in self.skip_in else dims[l + 1]
            lin = nn.Linear(dims[l], out_dim)
            if geometric_init:  # IGR / IDR geometric initialisation (network.py:49-63)
                if l == self.num_layers - 2:
                    nn.init.normal_(lin.weight, mean=np.sqrt(np.pi) / np.sqrt(dims[l]), std=0.0001)
                    nn.init.constant_(lin.bias, -bias)
                elif multires > 0 and l == 0:
                    nn.init.constant_(lin.bias, 0.0)
                    nn.init.constant_(lin.weight[:, 3:], 0.0)
                    nn.init.normal_(lin.weight[:, :3], 0.0, np.sqrt(2) / np.sqrt(out_dim))
                elif multires > 0 and l in self.skip_in:
                    nn.init.constant_(lin.bias, 0.0)
                    nn.init.normal_(lin.weight, 0.0, np.sqrt(2) / np.sqrt(out_dim))
                    nn.init.constant_(lin.weight[:, -(dims[0] - 3):], 0.0)
                else:
                    nn.init.constant_(lin.bias, 0.0)
                    nn.init.normal_(lin.weight, 0.0, np.sqrt(2) / np.sqrt(out_dim))
            if weight_norm:
                lin = nn.utils.weight_norm(lin)
            setattr(self, "lin" + str(l), lin)
        self.softplus = nn.Softplus(beta=100)
        self.rendcond = None
        self._cache = FoldCache()
        self._weff = None     # the layers' effective weights inside shared_weights()

    # ---- fused engine --------------------------------------------------------------------
    def _layers(self):
        out = []
        for l in range(self.num_layers - 1):
            lin = getattr(self, "lin" + str(l))
            if self.weight_norm:
                v, g = lin.weight_v, lin.weight_g
            else:
                v, g = lin.weight, None
            out.append(dict(v=v, g=g, b=lin.bias,
                            act=SR_ACT_SOFTPLUS100 if l < self.num_layers - 2 else SR_ACT_NONE,
                            skip=(l in self.skip_in)))
        return out

    def fused(self):
        layers = self._layers()
        params = [t for L in layers for t in (L["v"], L["g"], L["b"]) if t is not None]
        dev = params[0].device
        require_cuda(params[0], "ImplicitNetwork")
        if self.multires <= 0:
            raise RuntimeError("ImplicitNetwork: the fused engine expects multires > 0")

        def build():
            return ops.FusedMLP(3 + 6 * self.multires, self.multires, dev).fold(layers)

        return self._cache.get(params, build)

    def fused_sdf_only(self):
        net = self.fused()
        ex = self._cache.extra
        if "sdf_only" not in ex:
            ex["sdf_only"] = net.truncated_last(self.d_out)
        return ex["sdf_only"]

    def _pe_weights(self, ratio):
        return ops.annealing_weights(self.multires, ratio)

    def forward_fused(self, input, ratio, want_grad=False, want_feat=True, refine_about=0.0):
        """-> (sdf [P,d_out], grad [P,3] | None, feat | None) without building a graph.
        Large value-only batches run on the tensor-core engine; values within its error band of
        `refine_about` (the level a caller compares against: the MC balance value) are then re-evaluated
        on the fp32 engine so that the comparison's outcome is the fp32 one (None disables it)."""
        if self.d_out != 1:
            raise RuntimeError("ImplicitNetwork: fused path supports d_out == 1")
        r = ratio_value(ratio, "sdfRatio")
        nlast = getattr(self, "lin" + str(self.num_layers - 2)).bias.shape[0]
        nfeat = nlast - self.d_out if want_feat else 0
        net = self.fused() if nfeat > 0 else self.fused_sdf_only()
        w = self._pe_weights(r)
        net.set_pe_weights(w)
        pts = input.detach().reshape(-1, 3)
        if ops.TC_ENABLED and not want_grad and nfeat == 0 and pts.shape[0] >= ops.TC_MIN_POINTS:
            # large value-only batches (the 257^3 / 513^3 grid queries): tensor-core engine
            # (wgmma split-BF16 GEMM per layer, csrc/tc_gemm.cu)
            sdf = ops.tc_mlp_forward(net, pts, ch=1, n_out=1)
            if refine_about is not None:
                ops.sdf_refine_band(net, pts.contiguous().float(), sdf.view(-1), float(refine_about))
            return sdf.view(-1, 1), None, None
        sdf, grad, feat = ops.sdf_forward(net, pts, want_grad, nfeat)
        return sdf.view(-1, 1), grad, feat

    # ---- fused training path (tensor-core engine, forward tangents) --------------------------
    @contextlib.contextmanager
    def shared_weights(self):
        """Evaluations inside this context share ONE set of effective (weight-normed) weight tensors, i.e. one
        weight-norm sub-graph for several forward_train calls that are back-propagated together."""
        self._weff = self._weights()
        try:
            yield
        finally:
            self._weff = None

    def _weights(self):
        """The effective weight of every layer, in layer order."""
        from selfreconcode_b200 import train_ops as T
        lins = [getattr(self, "lin" + str(l)) for l in range(self.num_layers - 1)]
        return T.weight_norm_all(lins) if self.weight_norm else [lin.weight for lin in lins]

    def _effective(self, l):
        from selfreconcode_b200 import train_ops as T
        if self._weff is not None:
            return self._weff[l]
        lin = getattr(self, "lin" + str(l))
        return T.weight_norm_eff(lin.weight_v, lin.weight_g) if self.weight_norm else lin.weight

    def _train_ok(self):
        from selfreconcode_b200 import train_ops
        return train_ops.TC_TRAIN_ENABLED and self._fusable()

    def forward_train(self, input, ratio, want_grad=True, want_feat=True):
        """Differentiable (w.r.t. the input AND the parameters) evaluation on the tensor-core engine:
        -> (sdf [P,1], grad f [P,3] | None, feature [P,F] | None).  With want_grad the point travels as four
        rows (value + forward tangents), so grad f is an OUTPUT of the graph: losses on it (eikonal, normals)
        back-propagate with one reverse sweep -- the reference's create_graph=True / double backward
        (network.py:102-114, 608) without a second-order graph."""
        from selfreconcode_b200 import train_ops as T
        require_cuda(input, "ImplicitNetwork.forward_train")
        pts = input.reshape(-1, 3)
        P = pts.shape[0]
        ch = 4 if want_grad else 1
        L = self.num_layers - 1
        Ws, bs, acts, skips = [], [], [], []
        Weff = self._weff if self._weff is not None else self._weights()
        for l in range(L):
            lin = getattr(self, "lin" + str(l))
            W = Weff[l]
            b = lin.bias
            if l == L - 1 and not want_feat:      # value only: the feature head is not evaluated
                W, b = W[:self.d_out], b[:self.d_out]
            Ws.append(W)
            bs.append(b)
            acts.append(SR_ACT_SOFTPLUS100 if l < L - 1 else SR_ACT_NONE)
            skips.append(l in self.skip_in)
        d_in = 3 + 6 * self.multires
        x0 = T.embed_rows(pts, self.multires, self._pe_weights(ratio_value(ratio, "sdfRatio")), ch)
        packs = ops.tc_net(self.fused() if want_feat else self.fused_sdf_only()).layers
        out = T.tc_mlp(x0, T.MlpConfig(acts, skips, d_in, ch, packs), Ws, bs).view(P, ch, -1)
        sdf = out[:, 0, :self.d_out]
        grad = out[:, 1:, 0] if want_grad else None
        feat = out[:, 0, self.d_out:] if (want_feat and out.shape[2] > self.d_out) else None
        return sdf, grad, feat

    # ---- reference surface ---------------------------------------------------------------
    def _fusable(self):
        """The fused engines implement d_out == 1 with a positional encoding and layers at most 512 wide (the
        reference's getTmpSdf); other configurations (network.py:80,100) run the torch ops of _forward_autograd."""
        wide = max(getattr(self, "lin" + str(l)).bias.shape[0] for l in range(self.num_layers - 1))
        return self.multires > 0 and self.d_out == 1 and wide <= 512

    def forward(self, input, ratio):
        require_cuda(input, "ImplicitNetwork.forward")
        params_need = any(p.requires_grad for p in self.parameters())
        if self._fusable() and not needs_autograd(input) and not (torch.is_grad_enabled() and params_need):
            sdf, _, feat = self.forward_fused(input, ratio, False, True)
            self.rendcond = feat
            return sdf
        return self._forward_autograd(input, ratio)

    def _forward_autograd(self, input, ratio):
        ratio = ratio_value(ratio, "sdfRatio")
        if self.embed_fn is not None:
            if ratio is None:
                input = self.embed_fn(input)
            elif ratio <= 0:
                input = self.embed_fn(input, [0.0] * (self.multires * 2))
            else:
                ws = [w for w in self._pe_weights(ratio) for _ in (0, 1)]
                input = self.embed_fn(input, ws)
        x = input
        for l in range(self.num_layers - 1):
            lin = getattr(self, "lin" + str(l))
            if l in self.skip_in:
                x = torch.cat([x, input], 1) / np.sqrt(2)
            x = lin(x)
            if l < self.num_layers - 2:
                x = self.softplus(x)
        if x.shape[-1] > self.d_out:
            self.rendcond = x[:, self.d_out:]
            x = x[:, 0:self.d_out]
        else:
            self.rendcond = None
        return x

    def gradient(self, x, y=None):
        x.requires_grad_(True)
        if y is None:
            y = self.forward(x)
        d_output = torch.ones_like(y, requires_grad=False, device=y.device)
        gradients = torch.autograd.grad(outputs=y, inputs=x, grad_outputs=d_output,
                                        create_graph=True, retain_graph=True, only_inputs=True)[0]
        return gradients.view(-1, 3)


def getTmpSdf(device, multires, bias=0.6, feature_vector_size=256):
    net = ImplicitNetwork(feature_vector_size=feature_vector_size, d_in=3, d_out=1,
                          dims=[512] * 8, geometric_init=True, bias=bias, skip_in=[4],
                          weight_norm=True, multires=multires)
    return net.to(device)


def __getattr__(name):
    """`model.network.OptimNetwork` / `.getOptNet` (where the reference defines them, network.py:149,828)
    resolve to the orchestration module; looked up lazily because that module imports this one."""
    if name in ("OptimNetwork", "getOptNet"):
        from . import optim
        return getattr(optim, name)
    raise AttributeError(name)
