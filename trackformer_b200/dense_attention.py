"""Multi-head attention of the vanilla transformer on the hand-written dense-attention kernels (csrc/dense_attn.cu).

``mha_forward(module, query, key, value, key_padding_mask)`` evaluates an ``nn.MultiheadAttention`` module (sequence
first) with the same parameters (``in_proj_weight`` / ``in_proj_bias`` / ``out_proj``: the state_dict contract is
untouched) for the three calls of the reference's vanilla transformer (models/transformer.py):

* encoder self-attention   ``query = key = src + pos``, ``value = src``, key padding from the frame mask;
* decoder self-attention   ``query = key = tgt + query_pos``, ``value = tgt``;
* decoder cross-attention  ``query = tgt + query_pos``, ``key = memory + pos``, ``value = memory``, memory padding.

The packed in-projection is split over ``in_proj_weight`` / ``in_proj_bias`` (one [q | k] GEMM when ``query is key``),
the core ``dropout(softmax(q k^T / sqrt(32) + key_pad)) v`` is one launch forward and three backward on tensor cores
(split-TF32, fp32-level accuracy), and the output projection goes through ``fused_linear``.  Query and key lengths are
independent.  ``supported()`` is False -- and callers keep the stock module -- for CPU tensors, dtypes other than fp32,
head widths other than 32, and when ``TFB200_DENSE_ATTN=0``.

``need_weights=True`` also returns the attention probabilities averaged over heads, ``[B, Lq, Lk]`` (the stock
module's ``need_weights=True, average_attn_weights=True``): one more launch that re-forms them from the forward's q / k
and log-sum-exp (``dense_attention_weights``).  They are an inference output -- no gradient flows through them, and in
training with attention dropout (where the stock module returns the dropped-out weights) they are refused.
"""
from __future__ import annotations

import os

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ext, seeds
from .fused_linear import linear as fused_linear

_ENABLED = os.environ.get("TFB200_DENSE_ATTN", "1") != "0"


class _DenseAttention(Function):
    @staticmethod
    def forward(ctx, q, k, v, key_pad, seed, scale, keep_prob, need_weights=False):
        out, lse = ext.load().dense_attention_forward(q, k, v, key_pad, seed, scale, keep_prob)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.key_pad, ctx.seed, ctx.scale, ctx.keep_prob = key_pad, seed, scale, keep_prob
        ctx.need_weights = need_weights
        if not need_weights:
            return out
        weights = ext.load().dense_attention_weights(q, k, key_pad, lse, scale)
        ctx.mark_non_differentiable(weights)
        return out, weights

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out, grad_weights=None):
        q, k, v, out, lse = ctx.saved_tensors
        dq, dk, dv = ext.load().dense_attention_backward(q, k, v, ctx.key_pad, ctx.seed, out, lse, grad_out, ctx.scale,
                                                         ctx.keep_prob)
        return (dq, dk, dv, None, None, None, None) + ((None,) if ctx.need_weights else ())


def supported(module: torch.nn.MultiheadAttention, query: torch.Tensor) -> bool:
    e, h = module.embed_dim, module.num_heads
    return bool(_ENABLED and query.is_cuda and query.dtype == torch.float32 and e == 32 * h
                and module._qkv_same_embed_dim and module.in_proj_bias is not None and not module.batch_first
                and module.bias_k is None and not module.add_zero_attn)


def mha_forward(module: torch.nn.MultiheadAttention, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
                key_padding_mask=None, need_weights=False):
    """``module(query, key, value, key_padding_mask=..., need_weights=False)[0]`` for [L, B, E] inputs; with
    ``need_weights=True`` the pair ``(out, weights [B, Lq, Lk])``, the weights averaged over heads."""
    e, h = module.embed_dim, module.num_heads
    w, b = module.in_proj_weight, module.in_proj_bias
    if key is query:
        qk = fused_linear(query, w[:2 * e], b[:2 * e])              # [L, B, 2E]: q | k
        q, k = qk[..., :e], qk[..., e:]
    else:
        q = fused_linear(query, w[:e], b[:e])
        k = fused_linear(key, w[e:2 * e], b[e:2 * e])
    vv = fused_linear(value, w[2 * e:], b[2 * e:])
    p = float(module.dropout) if module.training else 0.0
    if need_weights and p > 0.0:
        raise NotImplementedError("dense_attention: need_weights=True is for inference; the attention weights after "
                                  "dropout are not formed (call module.eval() or set its dropout to 0)")
    seed = seeds.next_seed(query.device) if p > 0.0 else None
    key_pad = None
    if key_padding_mask is not None:
        key_pad = key_padding_mask if key_padding_mask.dtype == torch.bool else key_padding_mask != 0
    args = (q.unflatten(-1, (h, 32)), k.unflatten(-1, (h, 32)), vv.unflatten(-1, (h, 32)), key_pad, seed, 32 ** -0.5,
            1.0 - p)
    res = _DenseAttention.apply(*args, True) if need_weights else _DenseAttention.apply(*args)
    out = res[0] if need_weights else res
    out = fused_linear(out.flatten(2), module.out_proj.weight, module.out_proj.bias)
    return (out, res[1]) if need_weights else out


def attention(module: torch.nn.MultiheadAttention, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
              key_padding_mask=None, need_weights=False):
    """The attention output of ``module`` on the dense kernels where ``supported``, else the stock module's; with
    ``need_weights=True`` the pair ``(out, head-averaged weights [B, Lq, Lk])``."""
    if supported(module, query):
        return mha_forward(module, query, key, value, key_padding_mask, need_weights)
    out, weights = module(query, key, value, key_padding_mask=key_padding_mask, need_weights=need_weights)
    return (out, weights) if need_weights else out
