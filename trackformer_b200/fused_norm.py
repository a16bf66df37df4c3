"""``x = LayerNorm(x + dropout(branch))`` as one fused sm_90a kernel per direction.

Replaces the three-op forward / four-op backward chain the reference's transformer layers execute for every
residual connection (src/trackformer/models/deformable_transformer.py:284-285, 291-292, 360-361, 370-371,
377-378).  Same arithmetic (biased variance, eps inside the rsqrt, inverted dropout scaling 1/(1-p)); the
dropout mask is drawn with torch's generator (graph-capture safe) and consumed by the kernel.
CUDA only -- on other devices / unsupported widths it defers to the stock PyTorch ops of the wrapped modules
(that is the same arithmetic, not a different implementation of the MSDeformAttn core).
"""
from __future__ import annotations

import os

import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ext, seeds

# mask-free dropout (hash of a per-call device seed and the element index, like fused_linear.relu_dropout) instead of a
# bernoulli_ mask tensor per call; TFB200_LN_SEEDED=0 keeps the mask route
_SEEDED = os.environ.get("TFB200_LN_SEEDED", "1") != "0"


class _AddDropoutLayerNormSeeded(Function):
    @staticmethod
    def forward(ctx, x, branch, gamma, beta, p, eps):
        keep = 1.0 - p
        seed = seeds.next_seed(x.device)
        y, s, mean, rstd = ext.load().add_dropout_layernorm_seeded_forward(x, branch, seed, gamma, beta, keep, eps)
        ctx.save_for_backward(s, mean, rstd, gamma, seed)
        ctx.keep = keep
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        s, mean, rstd, gamma, seed = ctx.saved_tensors
        dx, dbranch, dgamma, dbeta = ext.load().add_dropout_layernorm_seeded_backward(dy, s, seed, gamma, mean, rstd,
                                                                                      ctx.keep)
        return dx, dbranch, dgamma, dbeta, None, None


class _AddDropoutLayerNorm(Function):
    @staticmethod
    def forward(ctx, x, branch, gamma, beta, p, training, eps):
        m = ext.load()
        keep = 1.0 - p
        mask = None
        if training and p > 0.0:
            mask = torch.empty(x.shape, dtype=torch.bool, device=x.device).bernoulli_(keep)
        y, s, mean, rstd = m.add_dropout_layernorm_forward(x, branch, mask, gamma, beta, keep, eps)
        ctx.save_for_backward(s, mean, rstd, gamma, mask)
        ctx.keep = keep
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        s, mean, rstd, gamma, mask = ctx.saved_tensors
        dx, dbranch, dgamma, dbeta = ext.load().add_dropout_layernorm_backward(dy, s, mask, gamma, mean, rstd, ctx.keep)
        return dx, dbranch, dgamma, dbeta, None, None, None


def supported(x: torch.Tensor, norm: nn.LayerNorm) -> bool:
    c = x.shape[-1]
    return (x.is_cuda and x.dtype == torch.float32 and c % 4 == 0 and c <= 512
            and norm.elementwise_affine and tuple(norm.normalized_shape) == (c,))


def add_dropout_layernorm(x: torch.Tensor, branch: torch.Tensor, dropout: nn.Dropout, norm: nn.LayerNorm) -> torch.Tensor:
    """``norm(x + dropout(branch))`` -- fused when the geometry allows, the module chain otherwise."""
    if supported(x, norm) and branch.shape == x.shape:
        if _SEEDED and dropout.training and dropout.p > 0.0:
            return _AddDropoutLayerNormSeeded.apply(x, branch, norm.weight, norm.bias, float(dropout.p), float(norm.eps))
        return _AddDropoutLayerNorm.apply(x, branch, norm.weight, norm.bias, float(dropout.p),
                                          bool(dropout.training), float(norm.eps))
    return norm(x + dropout(branch))
