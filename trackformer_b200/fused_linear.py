"""Linear layers and the FFN activation of the encoder with fused sm_90a epilogue kernels.

* ``linear(x, weight, bias)`` -- ``F.linear`` whose backward computes the bias gradient with the library's
  streaming column-sum kernel (one HBM-bound pass, deterministic) instead of PyTorch's generic reduction
  (33-40 us per [22223, 256..1024] call, 36 calls per C2 step).  The two GEMMs stay on cuBLAS tensor cores.
* ``relu_dropout(a, dropout)`` -- ``dropout(relu(a))`` in one pass, mask-free (the keep decision is a hash of a
  per-call seed and the element index; the backward reads the output only).

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


# Which of the three products run on it ("f" forward, "d" dgrad, "w" wgrad).  Measured on an H100 80GB HBM3 (400 W power
# limit, tools/gemm_bench.py): the split-token wgrad is within 1-7 % of the library (36.4 vs 35.3 us for
# 256 x 256 x 22223, 42.4 vs 39.6 us for 384 x 256); forward and dgrad are on par for N = 256 / 384 and up to 1.5x slower
# for the 1024-wide FFN products.  Default: only the wgrad runs on the hand-written kernel.
_TCGEN05_PARTS = os.environ.get("TFB200_TCGEN05_PARTS", "w")


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
