"""Segmentation heads of the deformable detector: ``DeformableDETRSegm`` and ``DeformableDETRSegmTracking``.

Mirror of src/trackformer/models/detr_segmentation.py:29-253 for the deformable classes: same class layout
(``DETRSegmBase`` mixed in front of ``DETRTrackingBase`` / ``DeformableDETR``, so the previous-frame forwards of tracking
training run without the mask head), constructor arguments, ``freeze_detr``, initialisation and parameter names
(``bbox_attention.{q,k}_linear.*``, ``mask_head.{lay1..5,gn1..5,out_lay,adapter1..3}.*``), and ``pred_masks``
``[B, Q, H/4, W/4]`` logits.

The reference's ``forward(samples, targets)`` lacks the ``prev_features`` argument its tracker passes
(tracker.py:306); here it is accepted and passed through.

On CPU tensors and in other dtypes the head runs the reference's torch ops.  On CUDA fp32 the convolutions stay in
cuDNN (channels-last) and everything between them is csrc/mask_head.cu.  The reference convolves ``cat(_expand(src, Q), bbox_mask)`` in
``lay1`` -- one copy of the image's 256-channel map per query -- and adds expanded adapter outputs; here ``lay1`` is
split by linearity into a per-image convolution of ``src`` and a per-query convolution of the attention maps,
and both per-image terms enter the fused GroupNorm / upsample-add kernels as operands broadcast over the queries.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn.functional as F
from torch import Tensor, nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ext
from .deformable_detr import DeformableDETR
from .detr_tracking import DETRTrackingBase
from .fused_linear import linear as fused_linear
from .util import NestedTensor


# ---------------------------------------------------------------------------------------------------------------------
class _MaskAttn(Function):
    @staticmethod
    def forward(ctx, q, k, pad, heads, scale):
        w = ext.load().mask_attn_forward(q, k, pad, heads, scale)
        ctx.save_for_backward(q.contiguous(), k.contiguous(), w)
        ctx.scale = scale
        return w

    @staticmethod
    @once_differentiable
    def backward(ctx, dw):
        q, k, w = ctx.saved_tensors
        dq, dk = ext.load().mask_attn_backward(q, k, w, dw, ctx.scale)
        return dq, dk, None, None, None


class _GroupNormReLU(Function):
    @staticmethod
    def forward(ctx, x, addend, gamma, beta, groups, per_image, eps):
        y, mean, rstd = ext.load().group_norm_relu_forward(x, addend, gamma, beta, groups, per_image, eps)
        ctx.save_for_backward(x, addend, y, gamma, mean, rstd)
        ctx.per_image = per_image
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, addend, y, gamma, mean, rstd = ctx.saved_tensors
        dx, da, dgamma, dbeta = ext.load().group_norm_relu_backward(dy, x, addend, y, gamma, mean, rstd, ctx.per_image)
        return dx, (da if addend is not None else None), dgamma, dbeta, None, None, None


class _UpsampleAdd(Function):
    @staticmethod
    def forward(ctx, x, a):
        ctx.geom = (a.shape[0], x.shape[2], x.shape[3])
        return ext.load().upsample_add_forward(x, a)

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        dx, da = ext.load().upsample_add_backward(dout, *ctx.geom)
        return dx, da


def group_norm_relu(x: Tensor, gn: nn.GroupNorm, addend: Optional[Tensor] = None, per_image: int = 1) -> Tensor:
    """``relu(gn(x + addend[n // per_image]))`` on channels-last CUDA fp32 maps (csrc/mask_head.cu)."""
    cl = torch.channels_last
    if addend is not None:
        addend = addend.contiguous(memory_format=cl)
    return _GroupNormReLU.apply(x.contiguous(memory_format=cl), addend, gn.weight, gn.bias, gn.num_groups, per_image,
                                float(gn.eps))


def upsample_add(x: Tensor, a: Tensor) -> Tensor:
    """``a[n // per_image] + F.interpolate(x, size=a.shape[-2:], mode="nearest")`` (csrc/mask_head.cu)."""
    cl = torch.channels_last
    return _UpsampleAdd.apply(x.contiguous(memory_format=cl), a.contiguous(memory_format=cl))


def mask_attention(q: Tensor, k: Tensor, pad: Optional[Tensor], heads: int, scale: float) -> Tensor:
    """softmax over positions of ``scale * q . k`` per head: q [B, Q, D], k [B, HW, D] -> [B, Q, heads, HW]."""
    return _MaskAttn.apply(q, k, pad, heads, scale)


# ---------------------------------------------------------------------------------------------------------------------
def _expand(tensor, length: int):
    return tensor.unsqueeze(1).repeat(1, int(length), 1, 1, 1).flatten(0, 1)


class MaskHeadSmallConv(nn.Module):
    """Convolutional head with group norm; FPN-style upsampling to stride 4 (detr_segmentation.py:111-197)."""

    def __init__(self, dim, fpn_dims, context_dim):
        super().__init__()
        inter_dims = [dim, context_dim // 2, context_dim // 4, context_dim // 8, context_dim // 16, context_dim // 64]
        self.lay1 = torch.nn.Conv2d(dim, dim, 3, padding=1)
        self.gn1 = torch.nn.GroupNorm(8, dim)
        self.lay2 = torch.nn.Conv2d(dim, inter_dims[1], 3, padding=1)
        self.gn2 = torch.nn.GroupNorm(8, inter_dims[1])
        self.lay3 = torch.nn.Conv2d(inter_dims[1], inter_dims[2], 3, padding=1)
        self.gn3 = torch.nn.GroupNorm(8, inter_dims[2])
        self.lay4 = torch.nn.Conv2d(inter_dims[2], inter_dims[3], 3, padding=1)
        self.gn4 = torch.nn.GroupNorm(8, inter_dims[3])
        self.lay5 = torch.nn.Conv2d(inter_dims[3], inter_dims[4], 3, padding=1)
        self.gn5 = torch.nn.GroupNorm(8, inter_dims[4])
        self.out_lay = torch.nn.Conv2d(inter_dims[4], 1, 3, padding=1)

        self.dim = dim

        self.adapter1 = torch.nn.Conv2d(fpn_dims[0], inter_dims[1], 1)
        self.adapter2 = torch.nn.Conv2d(fpn_dims[1], inter_dims[2], 1)
        self.adapter3 = torch.nn.Conv2d(fpn_dims[2], inter_dims[3], 1)

        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_uniform_(m.weight, a=1)
                nn.init.constant_(m.bias, 0)

    def _stages(self):
        return ((self.adapter1, self.lay3, self.gn3), (self.adapter2, self.lay4, self.gn4),
                (self.adapter3, self.lay5, self.gn5))

    def forward(self, x: Tensor, bbox_mask: Tensor, fpns: List[Tensor]):
        """x [B, C, H, W] per image, bbox_mask [B, Q, heads, H, W], fpns per image -> [B * Q, 1, H4, W4]"""
        if x.is_cuda and x.dtype == torch.float32:
            return self._forward_cuda(x, bbox_mask, fpns)
        x = torch.cat([_expand(x, bbox_mask.shape[1]), bbox_mask.flatten(0, 1)], 1)
        x = F.relu(self.gn1(self.lay1(x)))
        x = F.relu(self.gn2(self.lay2(x)))
        for (adapter, lay, gn), fpn in zip(self._stages(), fpns):
            cur_fpn = adapter(fpn)
            if cur_fpn.size(0) != x.size(0):
                cur_fpn = _expand(cur_fpn, x.size(0) // cur_fpn.size(0))
            x = cur_fpn + F.interpolate(x, size=cur_fpn.shape[-2:], mode="nearest")
            x = F.relu(gn(lay(x)))
        return self.out_lay(x)

    def _forward_cuda(self, x, bbox_mask, fpns):
        cl = torch.channels_last
        n_q = bbox_mask.shape[1]
        n_src = x.shape[1]
        # lay1(cat(_expand(x), bbox_mask)) = conv(x, W[:, :n_src]) + b (per image) + conv(bbox_mask, W[:, n_src:]) (per query)
        per_image = F.conv2d(x.contiguous(memory_format=cl), self.lay1.weight[:, :n_src], self.lay1.bias, padding=1)
        y = F.conv2d(bbox_mask.flatten(0, 1).contiguous(memory_format=cl), self.lay1.weight[:, n_src:], None, padding=1)
        y = group_norm_relu(y, self.gn1, per_image, n_q)
        y = group_norm_relu(self.lay2(y), self.gn2)
        for (adapter, lay, gn), fpn in zip(self._stages(), fpns):
            y = upsample_add(y, adapter(fpn.contiguous(memory_format=cl)))
            y = group_norm_relu(lay(y), gn)
        return self.out_lay(y)


class MHAttentionMap(nn.Module):
    """Attention softmax of the queries over a 2-d map, without the value product (detr_segmentation.py:200-216)."""

    def __init__(self, query_dim, hidden_dim, num_heads, dropout=0.0, bias=True):
        super().__init__()
        self.num_heads = num_heads
        self.hidden_dim = hidden_dim
        self.dropout = nn.Dropout(dropout)

        self.q_linear = nn.Linear(query_dim, hidden_dim, bias=bias)
        self.k_linear = nn.Linear(query_dim, hidden_dim, bias=bias)

        nn.init.zeros_(self.k_linear.bias)
        nn.init.zeros_(self.q_linear.bias)
        nn.init.xavier_uniform_(self.k_linear.weight)
        nn.init.xavier_uniform_(self.q_linear.weight)
        self.normalize_fact = float(hidden_dim / self.num_heads) ** -0.5

    def forward(self, q, k, mask: Optional[Tensor] = None):
        """q [B, Q, D], k [B, D, H, W] (may be a view of token-major memory), mask [B, H, W] -> [B, Q, heads, H, W]"""
        if q.is_cuda and q.dtype == torch.float32:
            b, _, h, w = k.shape
            k_tok = k.permute(0, 2, 3, 1).reshape(b, h * w, k.shape[1])     # a view of token-major encoder memory
            qp = fused_linear(q, self.q_linear.weight, self.q_linear.bias).contiguous()
            kp = fused_linear(k_tok, self.k_linear.weight, self.k_linear.bias).contiguous()
            pad = None if mask is None else mask.reshape(b, h * w)
            weights = mask_attention(qp, kp, pad, self.num_heads, self.normalize_fact)
            return self.dropout(weights.view(b, q.shape[1], self.num_heads, h, w))
        q = self.q_linear(q)
        k = F.conv2d(k, self.k_linear.weight.unsqueeze(-1).unsqueeze(-1), self.k_linear.bias)
        qh = q.view(q.shape[0], q.shape[1], self.num_heads, self.hidden_dim // self.num_heads)
        kh = k.view(k.shape[0], self.num_heads, self.hidden_dim // self.num_heads, k.shape[-2], k.shape[-1])
        weights = torch.einsum("bqnc,bnchw->bqnhw", qh * self.normalize_fact, kh)
        if mask is not None:
            weights.masked_fill_(mask.unsqueeze(1).unsqueeze(1), float("-inf"))
        weights = F.softmax(weights.flatten(2), dim=-1).view_as(weights)
        return self.dropout(weights)


# ---------------------------------------------------------------------------------------------------------------------
class DETRSegmBase(nn.Module):
    def __init__(self, freeze_detr=False):
        # like the reference this runs AFTER the detector's __init__ and must not call nn.Module.__init__
        if freeze_detr:
            for param in self.parameters():
                param.requires_grad_(False)

        nheads = self.transformer.nhead
        self.bbox_attention = MHAttentionMap(self.hidden_dim, self.hidden_dim, nheads, dropout=0.0)
        self.mask_head = MaskHeadSmallConv(self.hidden_dim + nheads, self.fpn_channels, self.hidden_dim)

    def forward(self, samples: NestedTensor, targets: list = None, prev_features=None):
        out, targets, features, memory, hs = super().forward(samples, targets, prev_features)

        src, mask = features[-2].decompose()                     # stride 16 (layer3)
        batch_size = src.shape[0]
        src = self.input_proj[-3](src)
        if mask.shape[-2:] != src.shape[-2:]:
            mask = F.interpolate(mask[None].float(), size=src.shape[-2:]).to(torch.bool)[0]
        fpns = [features[-2].tensors, features[-3].tensors, features[-4].tensors]

        bbox_mask = self.bbox_attention(hs[-1], memory[-3], mask=mask)
        seg_masks = self.mask_head(src, bbox_mask, fpns)
        out["pred_masks"] = seg_masks.view(batch_size, hs.shape[2], seg_masks.shape[-2], seg_masks.shape[-1])
        return out, targets, features, memory, hs


class DeformableDETRSegm(DETRSegmBase, DeformableDETR):
    def __init__(self, mask_kwargs, detr_kwargs):
        DeformableDETR.__init__(self, **detr_kwargs)
        DETRSegmBase.__init__(self, **mask_kwargs)


class DeformableDETRSegmTracking(DETRSegmBase, DETRTrackingBase, DeformableDETR):
    def __init__(self, mask_kwargs, tracking_kwargs, detr_kwargs):
        DeformableDETR.__init__(self, **detr_kwargs)
        DETRTrackingBase.__init__(self, **tracking_kwargs)
        DETRSegmBase.__init__(self, **mask_kwargs)


class PostProcessSegm(nn.Module):
    """Mask probabilities / binary masks at the original image sizes (detr_segmentation.py:219-253)."""

    def __init__(self, threshold=0.5):
        super().__init__()
        self.threshold = threshold

    @torch.no_grad()
    def forward(self, results, outputs, orig_target_sizes, max_target_sizes, return_probs=False, results_mask=None):
        assert len(orig_target_sizes) == len(max_target_sizes)
        max_h, max_w = max_target_sizes.max(0)[0].tolist()
        outputs_masks = outputs["pred_masks"].squeeze(2)
        outputs_masks = F.interpolate(outputs_masks, size=(max_h, max_w), mode="bilinear", align_corners=False)
        outputs_masks = outputs_masks.sigmoid().cpu()
        if not return_probs:
            outputs_masks = outputs_masks > self.threshold

        for i, (cur_mask, t, tt) in enumerate(zip(outputs_masks, max_target_sizes, orig_target_sizes)):
            img_h, img_w = t[0], t[1]
            masks = cur_mask[:, :img_h, :img_w].unsqueeze(1)
            masks = F.interpolate(masks.float(), size=tuple(tt.tolist()), mode="nearest")
            if not return_probs:
                masks = masks.byte()
            if results_mask is not None:
                masks = masks[results_mask[i]]
            results[i]["masks"] = masks
        return results
