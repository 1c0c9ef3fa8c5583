"""Glue between nn.Module parameters and the fused engine (ops.FusedMLP)."""
import torch

from selfreconcode_b200 import ops
from selfreconcode_b200._lib import SR_ACT_NONE, SR_ACT_SOFTPLUS100, SR_ACT_RELU, SR_ACT_TANH


def ratio_value(ratio, key):
    if isinstance(ratio, dict):
        return ratio[key]
    return ratio


def needs_autograd(*tensors):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


class _IndexRows(torch.autograd.Function):
    """t.index_select(0, idx) whose backward sums the rows of each index in a fixed order (index_put with accumulate,
    sorted by index on CUDA) instead of index_select's atomicAdd: a step's per-frame gradients (poses, translations,
    latent codes) are then bit-identical from run to run.  The backward is itself differentiable."""

    @staticmethod
    def forward(ctx, t, idx):
        ctx.save_for_backward(idx)
        ctx.n = t.shape[0]
        return t.index_select(0, idx)

    @staticmethod
    def backward(ctx, g):
        idx, = ctx.saved_tensors
        return scatter_rows(g, idx, ctx.n), None


def index_rows(t, idx):
    """Rows idx of t (dim 0), deterministic in the backward."""
    return _IndexRows.apply(t, idx)


def scatter_rows(src, idx, n):
    """[n, ...] with out[i] = sum of the rows src[j] with idx[j] == i, summed in a fixed order (differentiable)."""
    return src.new_zeros((n,) + tuple(src.shape[1:])).index_put((idx,), src, accumulate=True)


def require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError("%s: CUDA tensor required -- selfrecon_b200 has no CPU path" % what)


class FoldCache:
    """Re-folds (weight-norm, transpose, pad) when any parameter changed in place or was
    replaced; optimiser steps bump Tensor._version, load_state_dict copies in place too."""

    def __init__(self):
        self.sig = None
        self.net = None
        self.extra = {}

    def get(self, params, builder):
        sig = tuple((p.data_ptr(), p._version, str(p.device)) for p in params)
        if sig != self.sig:
            same_storage = self.sig is not None and self.net is not None and \
                tuple((a[0], a[2]) for a in sig) == tuple((a[0], a[2]) for a in self.sig)
            if same_storage and hasattr(self.net, "refold"):
                # only the VALUES changed (optimizer.step(), load_state_dict): refold into the same device buffers
                # -- descriptors, tensor-core packs, truncated views and captured graphs stay valid
                self.net.refold()
            else:
                self.net = builder()
                self.extra = {}
            self.sig = sig
        return self.net
