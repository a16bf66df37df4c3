"""Linear layers and the FFN activation of the encoder with fused sm_90a epilogue kernels.

* ``linear(x, weight, bias)`` -- ``F.linear`` whose backward computes the bias gradient with the library's
  streaming column-sum kernel (one HBM-bound pass, deterministic) instead of PyTorch's generic reduction
  (33-40 us per [22223, 256..1024] call, 36 calls per C2 step).  On the long-token TF32 route the products listed in
  _TCGEN05_PARTS run on the hand-written wgmma kernel (csrc/tf32_gemm.cu), the others on cuBLAS.
* ``relu_dropout(a, dropout)`` -- ``dropout(relu(a))`` in one pass, mask-free (the keep decision is a hash of a
  per-call seed and the element index; the backward reads the output only).
* ``ffn(x, linear1, linear2, dropout)`` -- the encoder FFN ``linear2(dropout(relu(linear1(x))))`` on the long-token
  TF32 route, with the ReLU-dropout and its gradient in the epilogues of the hand-written GEMM (``ffn_fusable`` says
  when it applies).

Both defer to the stock PyTorch ops on CPU tensors and for shapes outside the kernels' domain -- the same arithmetic,
not an alternative implementation of the MSDeformAttn core.  Reference call sites:
src/trackformer/models/deformable_transformer.py:282-286 (FFN), ops/modules/ms_deform_attn.py:64-88 (projections).
"""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ext, seeds

_MIN_ROWS = 64            # from here on the column-sum kernels beat the generic reduction (single launch up to 2048 rows)
_SPLIT_K = os.environ.get("TFB200_WGRAD_SPLITK", "0") == "1"      # opt-in: see weight_grad


def weight_grad(gy2: torch.Tensor, x2: torch.Tensor) -> torch.Tensor:
    """dW = gy2^T @ x2 for a long token axis ([22223, C] operands at the benchmark size).

    The product is a small [c_out, c_in] tile grid reduced over tens of thousands of rows; the library GEMM does not
    split that reduction and runs 16-64 CTAs on a 132-SM part.  Splitting
    the token axis into `s` slabs turns it into one batched GEMM with s x as many CTAs plus a [s, c_out, c_in] sum:
    same products, fp32 accumulation, only the summation order over tokens changes.

    It is OFF unless TFB200_WGRAD_SPLITK=1: inside the replayed training step the operands were just written and sit
    in L2, and the three launches cost more than the split saves (tools/wgrad_bench.py times both)."""
    k, c_out = gy2.shape
    c_in = x2.shape[1]
    tiles = -(-c_out // 128) * -(-c_in // 128)
    sms = torch.cuda.get_device_properties(gy2.device).multi_processor_count if gy2.is_cuda else 1
    splits = min(16, max(1, (2 * sms) // (3 * tiles)), k // 1024)
    if not _SPLIT_K or splits < 2 or not (gy2.is_contiguous() and x2.is_contiguous()):
        return gy2.t() @ x2
    slab = (k // splits) & ~7
    main = slab * splits
    gw = torch.bmm(gy2[:main].view(splits, slab, c_out).transpose(1, 2), x2[:main].view(splits, slab, c_in)).sum(0)
    if main < k:
        gw.addmm_(gy2[main:].t(), x2[main:])
    return gw


# Forward products of the long-token Linears on the hand-written wgmma kernel (csrc/tf32_gemm.cu) whenever TF32
# tensor-core math is allowed (torch.backends.cuda.matmul.allow_tf32 -- the benchmark setting; strict-fp32 runs keep the
# library's fp32 GEMM).  TFB200_TCGEN05_LINEAR=0 switches it off (A/B timing).
_TCGEN05 = os.environ.get("TFB200_TCGEN05_LINEAR", "1") != "0"


# Which of the three products run on it ("f" forward, "d" dgrad, "w" wgrad).  Measured on an H100 80GB HBM3 (700 W power
# limit, tools/gemm_bench.py, L2 flushed, us ours / library, M = 22223 tokens, K -> N):
#   256 -> 256    forward 30.1 / 28.8   dgrad 30.8 / 32.9   wgrad 36.2 / 35.6
#   256 -> 384    forward 35.1 / 32.5   dgrad 36.9 / 41.1   wgrad 43.2 / 40.3
#   256 -> 1024   forward 74.7 / 56.0   dgrad 67.3 / 83.3   wgrad 83.7 / 83.1
#   1024 -> 256   forward 66.6 / 62.8   dgrad 75.7 / 80.0   wgrad 83.9 / 82.8
# The dgrad (the forward kernel on the transposed weight) is faster than the library on every long-token shape, the
# forward is not, the wgrad is on par.  Default: dgrad and wgrad on the hand-written kernel.  The FFN's first forward
# product and second dgrad always run on it when the FFN takes the fused route (ffn below).
_TCGEN05_PARTS = os.environ.get("TFB200_TCGEN05_PARTS", "dw")


def _tcgen05_ok(x, weight):
    if not (_TCGEN05 and torch.backends.cuda.matmul.allow_tf32 and x.is_contiguous() and weight.is_contiguous()):
        return False
    rows = x.numel() // x.shape[-1]
    if rows < 2048:                      # decoder-sized products: the library is as fast (gemm_bench, M = 300)
        return False
    return bool(ext.load().tf32_linear_supported(rows, weight.shape[0], weight.shape[1]))


class _LinearColsum(Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        ctx.tc = _tcgen05_ok(x, weight)
        if ctx.tc and "f" in _TCGEN05_PARTS:
            return ext.load().tf32_linear(x, weight, bias, False)
        return F.linear(x, weight, bias)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        gy2 = gy.reshape(-1, gy.shape[-1])
        gx = gw = gb = None
        m = ext.load()
        if ctx.needs_input_grad[0]:
            if ctx.tc and "d" in _TCGEN05_PARTS and gy2.is_contiguous():
                gx = m.tf32_linear_dgrad(gy2, weight).view(x.shape)
            else:
                gx = (gy2 @ weight).view(x.shape)
        if ctx.needs_input_grad[1]:
            if ctx.tc and "w" in _TCGEN05_PARTS and gy2.is_contiguous():
                gw = m.tf32_linear_wgrad(gy2, x.reshape(-1, x.shape[-1]))
            else:
                gw = weight_grad(gy2, x.reshape(-1, x.shape[-1]))
        if ctx.needs_input_grad[2]:
            gb = ext.load().colsum(gy2)
        return gx, gw, gb


def linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    rows = x.numel() // x.shape[-1]
    c_out = weight.shape[0]
    if (x.is_cuda and x.dtype == torch.float32 and bias is not None and rows >= _MIN_ROWS
            and c_out % 4 == 0 and c_out <= 1024 and torch.is_grad_enabled()):
        return _LinearColsum.apply(x, weight, bias)
    return F.linear(x, weight, bias)


class _ReluDropout(Function):
    @staticmethod
    def forward(ctx, a, p, training):
        m = ext.load()
        keep = 1.0 - p
        seed = None
        if training:
            seed = seeds.next_seed(a.device)
        h = m.relu_dropout_forward(a, seed, keep, training)
        ctx.save_for_backward(h)
        ctx.keep, ctx.training = keep, training
        return h

    @staticmethod
    @once_differentiable
    def backward(ctx, gh):
        (h,) = ctx.saved_tensors
        return ext.load().relu_dropout_backward(gh, h, ctx.keep, ctx.training), None, None


def relu_dropout(a: torch.Tensor, dropout: nn.Dropout) -> torch.Tensor:
    """``dropout(relu(a))``."""
    if a.is_cuda and a.dtype == torch.float32 and a.numel() % 4 == 0 and a.numel() >= 8192:
        training = bool(dropout.training and dropout.p > 0.0)
        return _ReluDropout.apply(a, float(dropout.p), training)
    return dropout(F.relu(a))


def _weight_grad(gy2, x2):
    if "w" in _TCGEN05_PARTS:
        return ext.load().tf32_linear_wgrad(gy2, x2)
    return weight_grad(gy2, x2)


class _FFN(Function):
    """``linear2(dropout(relu(linear1(x))))`` with the activation in the GEMM epilogues: the forward's first product
    writes the activated hidden tensor h directly, and the backward's dgrad of the second product writes the gradient
    of the pre-activation (h > 0 ? g / keep : 0) directly.  At [22223, 1024] fp32 that removes one 182 MB elementwise
    pass from each direction.  The hidden tensor's mask is relu_dropout's (same hash, same flat index)."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, p, training):
        m = ext.load()
        keep = 1.0 - p
        seed = seeds.next_seed(x.device) if training else None
        h = m.tf32_linear_relu_dropout(x, w1, b1, seed, keep, training)
        ff = m.tf32_linear(h, w2, b2, False) if "f" in _TCGEN05_PARTS else F.linear(h, w2, b2)
        ctx.save_for_backward(x, h, w1, w2)
        ctx.keep, ctx.training = keep, training
        return ff

    @staticmethod
    @once_differentiable
    def backward(ctx, gff):
        x, h, w1, w2 = ctx.saved_tensors
        m = ext.load()
        g2 = gff.reshape(-1, gff.shape[-1]).contiguous()
        h2 = h.reshape(-1, h.shape[-1])
        x2 = x.reshape(-1, x.shape[-1])
        ga = m.tf32_linear_dgrad_relu_dropout(g2, w2, h2, ctx.keep, ctx.training)
        gx = gw1 = gb1 = gw2 = gb2 = None
        if ctx.needs_input_grad[0]:
            gx = (m.tf32_linear_dgrad(ga, w1) if "d" in _TCGEN05_PARTS else ga @ w1).view(x.shape)
        if ctx.needs_input_grad[1]:
            gw1 = _weight_grad(ga, x2)
        if ctx.needs_input_grad[2]:
            gb1 = m.colsum(ga)
        if ctx.needs_input_grad[3]:
            gw2 = _weight_grad(g2, h2)
        if ctx.needs_input_grad[4]:
            gb2 = m.colsum(g2)
        return gx, gw1, gb1, gw2, gb2, None, None


def ffn_fusable(x: torch.Tensor, linear1: nn.Linear, linear2: nn.Linear, dropout: nn.Dropout) -> bool:
    """Whether ``ffn`` takes this FFN: the long-token TF32 training route (_tcgen05_ok: TF32 allowed, at least 2048
    rows, shapes the kernel tiles) with biases, fp32 CUDA tensors and a dropout probability below 1.  Strict-fp32
    runs, short token axes and no-grad calls keep the composition of ``linear`` and ``relu_dropout``."""
    w1, w2 = linear1.weight, linear2.weight
    if not (x.is_cuda and x.dtype == torch.float32 and w1.dtype == torch.float32 and w2.dtype == torch.float32
            and linear1.bias is not None and linear2.bias is not None and dropout.p < 1.0
            and torch.is_grad_enabled() and w2.is_contiguous() and _tcgen05_ok(x, w1)):
        return False
    return bool(ext.load().tf32_linear_supported(x.numel() // x.shape[-1], w2.shape[0], w2.shape[1]))


def ffn(x: torch.Tensor, linear1: nn.Linear, linear2: nn.Linear, dropout: nn.Dropout) -> torch.Tensor:
    """``linear2(dropout(relu(linear1(x))))`` as one autograd function (see _FFN); call when ``ffn_fusable``."""
    training = bool(dropout.training and dropout.p > 0.0)
    return _FFN.apply(x, linear1.weight, linear1.bias, linear2.weight, linear2.bias, float(dropout.p), training)
