"""Segmentation heads: ``DETRSegm``, ``DETRSegmTracking``, ``DeformableDETRSegm`` and ``DeformableDETRSegmTracking``.

Mirror of src/trackformer/models/detr_segmentation.py:29-253: same class layout
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

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor, nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ext
from .deformable_detr import DETR, DeformableDETR
from .detr_tracking import TWO_STAGE_TRACKING, DETRTrackingBase
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


class _MaskAttnRows(Function):
    @staticmethod
    def forward(ctx, q, k, pad, offsets, heads, scale):
        w = ext.load().mask_attn_rows_forward(q, k, pad, offsets, heads, scale)
        ctx.save_for_backward(q.contiguous(), k.contiguous(), offsets, w)
        ctx.scale = scale
        return w

    @staticmethod
    @once_differentiable
    def backward(ctx, dw):
        q, k, offsets, w = ctx.saved_tensors
        dq, dk = ext.load().mask_attn_rows_backward(q, k, offsets, w, dw, ctx.scale)
        return dq, dk, None, None, None, None


class _GroupNormReLURows(Function):
    @staticmethod
    def forward(ctx, x, addend, offsets, gamma, beta, groups, eps):
        y, mean, rstd = ext.load().group_norm_relu_rows_forward(x, addend, offsets, gamma, beta, groups, eps)
        ctx.save_for_backward(x, addend, offsets, y, gamma, mean, rstd)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, addend, offsets, y, gamma, mean, rstd = ctx.saved_tensors
        dx, da, dgamma, dbeta = ext.load().group_norm_relu_rows_backward(dy, x, addend, offsets, y, gamma, mean, rstd)
        return dx, da, None, dgamma, dbeta, None, None


class _UpsampleAddRows(Function):
    @staticmethod
    def forward(ctx, x, a, offsets):
        ctx.save_for_backward(offsets)
        ctx.geom = (x.shape[2], x.shape[3])
        return ext.load().upsample_add_rows_forward(x, a, offsets)

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        offsets, = ctx.saved_tensors
        dx, da = ext.load().upsample_add_rows_backward(dout, offsets, *ctx.geom)
        return dx, da, None


class RaggedRows:
    """Query rows owned unevenly by the images of a batch: image b owns rows ``offsets[b] .. offsets[b + 1]``.
    ``offsets`` int32 [B + 1] and ``image`` int64 [P] (row -> image) live on the device; ``sizes`` are the host counts
    they were built from, so nothing is read back."""

    def __init__(self, sizes, device):
        self.sizes = [int(n) for n in sizes]
        acc = [0]
        for n in self.sizes:
            acc.append(acc[-1] + n)
        self.offsets = torch.tensor(acc, dtype=torch.int32).to(device, non_blocking=True)
        self.image = torch.repeat_interleave(torch.arange(len(self.sizes)),
                                             torch.tensor(self.sizes, dtype=torch.long)).to(device, non_blocking=True)

    @property
    def total(self) -> int:
        return sum(self.sizes)


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
    """``scale * q . k`` per head, -inf where ``pad``, softmax over each query's heads and positions together (one
    partition sum per query, as MHAttentionMap's ``softmax(weights.flatten(2))``): q [B, Q, D], k [B, HW, D] ->
    [B, Q, heads, HW]."""
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

    def forward(self, x: Tensor, bbox_mask: Tensor, fpns: List[Tensor], rows: Optional[RaggedRows] = None):
        """x [B, C, H, W] per image, bbox_mask [B, Q, heads, H, W], fpns per image -> [B * Q, 1, H4, W4].
        With ``rows``: bbox_mask [P, heads, H, W], row p belonging to image ``rows.image[p]`` -> [P, 1, H4, W4]."""
        if x.is_cuda and x.dtype == torch.float32:
            if rows is not None:
                return self._forward_cuda_rows(x, bbox_mask, fpns, rows)
            return self._forward_cuda(x, bbox_mask, fpns)
        if rows is not None:
            x = torch.cat([x.index_select(0, rows.image), bbox_mask], 1)
            x = F.relu(self.gn1(self.lay1(x)))
            x = F.relu(self.gn2(self.lay2(x)))
            for (adapter, lay, gn), fpn in zip(self._stages(), fpns):
                cur_fpn = adapter(fpn).index_select(0, rows.image)
                x = cur_fpn + F.interpolate(x, size=cur_fpn.shape[-2:], mode="nearest")
                x = F.relu(gn(lay(x)))
            return self.out_lay(x)
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

    def _forward_cuda_rows(self, x, bbox_mask, fpns, rows):
        """``_forward_cuda`` over ragged rows: the per-image terms enter the ragged kernels, which broadcast them over
        each image's rows and sum their gradients over those rows."""
        cl = torch.channels_last
        n_src = x.shape[1]
        per_image = F.conv2d(x.contiguous(memory_format=cl), self.lay1.weight[:, :n_src], self.lay1.bias, padding=1)
        y = F.conv2d(bbox_mask.contiguous(memory_format=cl), self.lay1.weight[:, n_src:], None, padding=1)
        y = _GroupNormReLURows.apply(y.contiguous(memory_format=cl), per_image.contiguous(memory_format=cl),
                                     rows.offsets, self.gn1.weight, self.gn1.bias, self.gn1.num_groups,
                                     float(self.gn1.eps))
        y = group_norm_relu(self.lay2(y), self.gn2)
        for (adapter, lay, gn), fpn in zip(self._stages(), fpns):
            a = adapter(fpn.contiguous(memory_format=cl)).contiguous(memory_format=cl)
            y = _UpsampleAddRows.apply(y.contiguous(memory_format=cl), a, rows.offsets)
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

    def forward(self, q, k, mask: Optional[Tensor] = None, rows: Optional[RaggedRows] = None):
        """q [B, Q, D], k [B, D, H, W] (may be a view of token-major memory), mask [B, H, W] -> [B, Q, heads, H, W].
        With ``rows``: q [P, D], row p attending to image ``rows.image[p]`` -> [P, heads, H, W]."""
        if rows is not None:
            return self._forward_rows(q, k, mask, rows)
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

    def _forward_rows(self, q, k, mask, rows):
        b, _, h, w = k.shape
        if q.is_cuda and q.dtype == torch.float32:
            k_tok = k.permute(0, 2, 3, 1).reshape(b, h * w, k.shape[1])
            qp = fused_linear(q, self.q_linear.weight, self.q_linear.bias).contiguous()
            kp = fused_linear(k_tok, self.k_linear.weight, self.k_linear.bias).contiguous()
            pad = None if mask is None else mask.reshape(b, h * w)
            weights = _MaskAttnRows.apply(qp, kp, pad, rows.offsets, self.num_heads, self.normalize_fact)
            return self.dropout(weights.view(q.shape[0], self.num_heads, h, w))
        q = self.q_linear(q)
        k = F.conv2d(k, self.k_linear.weight.unsqueeze(-1).unsqueeze(-1), self.k_linear.bias)
        qh = q.view(q.shape[0], self.num_heads, self.hidden_dim // self.num_heads)
        kh = k.view(b, self.num_heads, self.hidden_dim // self.num_heads, h, w).index_select(0, rows.image)
        weights = torch.einsum("pnc,pnchw->pnhw", qh * self.normalize_fact, kh)
        if mask is not None:
            weights = weights.masked_fill(mask.index_select(0, rows.image).unsqueeze(1), float("-inf"))
        weights = F.softmax(weights.flatten(1), dim=-1).view_as(weights)
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

    def forward(self, samples: NestedTensor, targets: list = None, prev_features=None, prev_valid=None):
        out, targets, features, memory, hs = self.detect(samples, targets, prev_features, prev_valid)
        out["pred_masks"] = self.mask_logits(features, memory, hs)
        return out, targets, features, memory, hs

    def detect(self, samples: NestedTensor, targets: list = None, prev_features=None, prev_valid=None):
        """The detection forward without the mask head: ``forward``'s return value without ``pred_masks``."""
        return super().forward(samples, targets, prev_features, prev_valid)

    def mask_logits(self, features, memory, hs, rows=None) -> Tensor:
        """Mask logits ``[B, len(rows), H/4, W/4]`` of the query rows ``rows`` (all rows if None) from the outputs of
        ``detect``.  Every query has its own attention softmax and its own GroupNorm sample, so a row's logits do not
        depend on which other rows are computed with it.

        ``rows=(src, sizes)`` selects a different set of rows per image: image b contributes ``sizes[b]`` rows (host
        ints), ``src`` [sum(sizes)] (device) holds their query indices image after image.  The result is then the
        compact ``[sum(sizes), H/4, W/4]``: row i is the mask of query ``src[i]`` of its image (a training step's
        matched queries; nothing is read back from the device)."""
        return self.mask_logits_from(*self.mask_inputs(features, memory, hs), rows=rows)

    def mask_inputs(self, features, memory, hs):
        """What the mask branch reads from the detector: ``(queries [B, Q, D], memory map [B, D, h, w], src map
        [B, D, h, w], its pad mask [B, h, w], fpns)`` -- the last decoder layer, the attention keys, the per-image
        ``lay1`` input and the three FPN maps, for the deformable and the vanilla layout."""
        if isinstance(memory, list):                               # deformable: per-level memory, stride 16 (layer3)
            src, mask = features[-2].decompose()
            src = self.input_proj[-3](src)
            if mask.shape[-2:] != src.shape[-2:]:
                mask = F.interpolate(mask[None].float(), size=src.shape[-2:]).to(torch.bool)[0]
            fpns = [features[-2].tensors, features[-3].tensors, features[-4].tensors]
            memory = memory[-3]
        else:                                                      # vanilla DETR: stride-32 memory [B, C, h, w]
            src, mask = features[-1].decompose()
            src = self.input_proj(src)
            fpns = [features[2].tensors, features[1].tensors, features[0].tensors]
        return hs[-1], memory, src, mask, fpns

    def mask_logits_from(self, q, memory, src, mask, fpns, rows=None) -> Tensor:
        """``mask_logits`` from the outputs of ``mask_inputs``."""
        batch_size = src.shape[0]
        if isinstance(rows, tuple):
            src_rows, sizes = rows
            ragged = RaggedRows(sizes, q.device)
            if ragged.total == 0:
                h4, w4 = fpns[-1].shape[-2:]
                return q.new_zeros((0, h4, w4))
            flat = ragged.image * q.shape[1] + src_rows.to(device=q.device, dtype=torch.long)
            q = q.flatten(0, 1).index_select(0, flat)
            bbox_mask = self.bbox_attention(q, memory, mask=mask, rows=ragged)
            seg_masks = self.mask_head(src, bbox_mask, fpns, rows=ragged)
            return seg_masks.view(ragged.total, seg_masks.shape[-2], seg_masks.shape[-1])
        if rows is not None:
            q = q.index_select(1, torch.as_tensor(rows, dtype=torch.long, device=q.device))
        bbox_mask = self.bbox_attention(q, memory, mask=mask)
        seg_masks = self.mask_head(src, bbox_mask, fpns)
        return seg_masks.view(batch_size, q.shape[1], seg_masks.shape[-2], seg_masks.shape[-1])


class DETRSegm(DETRSegmBase, DETR):
    def __init__(self, mask_kwargs, detr_kwargs):
        DETR.__init__(self, **detr_kwargs)
        DETRSegmBase.__init__(self, **mask_kwargs)


class DETRSegmTracking(DETRSegmBase, DETRTrackingBase, DETR):
    def __init__(self, mask_kwargs, tracking_kwargs, detr_kwargs):
        DETR.__init__(self, **detr_kwargs)
        DETRTrackingBase.__init__(self, **tracking_kwargs)
        DETRSegmBase.__init__(self, **mask_kwargs)


class DeformableDETRSegm(DETRSegmBase, DeformableDETR):
    def __init__(self, mask_kwargs, detr_kwargs):
        DeformableDETR.__init__(self, **detr_kwargs)
        DETRSegmBase.__init__(self, **mask_kwargs)


class DeformableDETRSegmTracking(DETRSegmBase, DETRTrackingBase, DeformableDETR):
    def __init__(self, mask_kwargs, tracking_kwargs, detr_kwargs):
        if detr_kwargs.get("two_stage"):
            raise NotImplementedError(TWO_STAGE_TRACKING)
        DeformableDETR.__init__(self, **detr_kwargs)
        DETRTrackingBase.__init__(self, **tracking_kwargs)
        DETRSegmBase.__init__(self, **mask_kwargs)


def resolve_track_masks(logits: Tensor, src, ids, prev_label: Optional[Tensor], size, crop, orig) -> Tensor:
    """The online tracker's masks of one frame as a label map ``[H, W]`` int32 (track id, -1 for background).

    ``ids`` are the active tracks in list order; ``src[t]`` is the row of ``logits`` ``[K, h, w]`` (stride-4 mask
    logits) whose mask track ``t`` takes this frame, or -1 for a track that keeps its previous mask
    ``prev_label == ids[t]``.  Same values as the reference: ``PostProcessSegm(return_probs=True)`` (bilinear to
    ``size``, sigmoid, crop to ``crop``, nearest to ``orig``), stacked with the kept boolean masks as 0 / 1, and every
    pixel labelled with the first track of maximal value if that value exceeds 0.5 (models/tracker.py:509-521).

    On CUDA fp32 logits this is one launch of csrc/track_masks.cu; otherwise the reference's torch ops."""
    return resolve_track_masks_many([(logits, src, ids, prev_label, size, crop, orig)])[0]


def resolve_track_masks_many(jobs) -> List[Tensor]:
    """``resolve_track_masks`` of several frames (e.g. one per sequence of a multi-sequence step): ``jobs`` is a list
    of its argument tuples ``(logits, src, ids, prev_label, size, crop, orig)``; returns their label maps in order.

    When every job's logits are CUDA fp32 on one device, all of them are ONE launch of csrc/track_masks.cu (up to 16
    per launch), each label map equal bit for bit to its own call; otherwise each job takes the reference's torch ops."""
    jobs = list(jobs)
    if not jobs:
        return []
    dev = jobs[0][0].device
    if all(j[0].is_cuda and j[0].dtype == torch.float32 and j[0].device == dev for j in jobs):
        srcs, idss = [], []
        for _, src, ids, *_ in jobs:
            srcs.append(torch.as_tensor(src, dtype=torch.int32).reshape(-1).cpu().numpy())
            idss.append(torch.as_tensor(ids, dtype=torch.int32).reshape(-1).cpu().numpy())
        packed = torch.from_numpy(np.concatenate(srcs + idss).astype(np.int32)).to(dev, non_blocking=True)
        views, o = [], 0
        for a in srcs + idss:
            views.append(packed[o:o + len(a)])
            o += len(a)
        n = len(jobs)
        out = []
        for c in range(0, n, 16):
            part = range(c, min(c + 16, n))
            out += ext.load().track_masks_batched(
                [jobs[i][0].contiguous() for i in part], [views[i] for i in part], [views[n + i] for i in part],
                [None if jobs[i][3] is None else jobs[i][3].to(device=dev, dtype=torch.int32) for i in part],
                [[int(jobs[i][4][0]), int(jobs[i][4][1]), int(jobs[i][5][0]), int(jobs[i][5][1]),
                  int(jobs[i][6][0]), int(jobs[i][6][1])] for i in part])
        return out
    return [_resolve_track_masks_host(*job) for job in jobs]


def _resolve_track_masks_host(logits: Tensor, src, ids, prev_label: Optional[Tensor], size, crop, orig) -> Tensor:
    """``resolve_track_masks`` with the reference's torch ops (any device and dtype)."""
    H, W = (int(v) for v in orig)
    src = torch.as_tensor(src, dtype=torch.int32).reshape(-1)
    ids = torch.as_tensor(ids, dtype=torch.int32).reshape(-1)
    dev = logits.device
    if len(ids) == 0:
        return torch.full((H, W), -1, dtype=torch.int32, device=dev)
    fresh = src >= 0
    probs = torch.empty(len(ids), H, W, dtype=torch.float32, device=dev)
    if bool(fresh.any()):
        rows = logits.index_select(0, src[fresh].long().to(dev))
        p = F.interpolate(rows[None].float(), size=(int(size[0]), int(size[1])), mode="bilinear", align_corners=False)
        p = p.sigmoid()[0, :, :int(crop[0]), :int(crop[1])].unsqueeze(1)
        probs[fresh.to(dev)] = F.interpolate(p, size=(H, W), mode="nearest")[:, 0]
    if not bool(fresh.all()):
        stale_ids = ids[~fresh].to(dev)
        probs[(~fresh).to(dev)] = (prev_label.to(dev)[None] == stale_ids[:, None, None]).float()
    arg = probs.argmax(0)
    keep = probs.gather(0, arg[None])[0] > 0.5
    return torch.where(keep, ids.to(dev)[arg], torch.full_like(arg, -1, dtype=torch.int32)).to(torch.int32)


class PostProcessSegm(nn.Module):
    """Mask probabilities / binary masks at the original image sizes (detr_segmentation.py:219-253)."""

    def __init__(self, threshold=0.5):
        super().__init__()
        self.threshold = threshold

    @torch.no_grad()
    def forward(self, results, outputs, orig_target_sizes, max_target_sizes, return_probs=False, results_mask=None,
                masks_on_device=False):
        """`masks_on_device=True` keeps the masks where the model's outputs are, as bool (or the probabilities with
        `return_probs`), with the values of the default route: COCO mask evaluation then reads them in place."""
        assert len(orig_target_sizes) == len(max_target_sizes)
        max_h, max_w = max_target_sizes.max(0)[0].tolist()
        outputs_masks = outputs["pred_masks"].squeeze(2)
        outputs_masks = F.interpolate(outputs_masks, size=(max_h, max_w), mode="bilinear", align_corners=False)
        outputs_masks = outputs_masks.sigmoid()
        if not masks_on_device:
            outputs_masks = outputs_masks.cpu()
        if not return_probs:
            outputs_masks = outputs_masks > self.threshold

        for i, (cur_mask, t, tt) in enumerate(zip(outputs_masks, max_target_sizes, orig_target_sizes)):
            img_h, img_w = t[0], t[1]
            masks = cur_mask[:, :img_h, :img_w].unsqueeze(1)
            masks = F.interpolate(masks.float(), size=tuple(tt.tolist()), mode="nearest")
            if not return_probs:
                masks = masks.bool() if masks_on_device else masks.byte()
            if results_mask is not None:
                masks = masks[results_mask[i]]
            results[i]["masks"] = masks
        return results


def pillow_nearest_src(n_in: int, n_out: int) -> np.ndarray:
    """Source index of each of `n_out` outputs of Pillow's NEAREST resize from `n_in`: int(v), v = s / 2 then v += s
    accumulated in double, s = n_in / n_out (ImagingScaleAffine).  Not ATen's nearest index."""
    s = n_in / n_out
    steps = np.full(n_out, s, np.float64)
    steps[0] = s / 2
    return np.add.accumulate(steps).astype(np.int64)


PANOPTIC_SIGMOID = ("panoptic post-processing needs a softmax classifier: PostProcessPanoptic takes a softmax over the "
                    "class logits and treats the last column as 'no object', so on a sigmoid (focal-loss) head it would "
                    "silently drop the last real class")


class PostProcessPanoptic(nn.Module):
    """The model's outputs as COCO panoptic results (detr_segmentation.py:256-388): one dict per image,
    ``{"png_string": bytes, "segments_info": [{"id", "isthing", "category_id", "area"}]}``.

    The reference's semantics, quirks included: kept queries are ``argmax != last and max softmax > threshold``; their
    padded stride-4 logits are bilinearly upsampled straight to the unpadded processed size; every pixel takes the
    first kept query of maximal softmax; on the first pass the later queries of a stuff class merge into its first; the
    map is resized to the target size with Pillow's NEAREST; while any segment has an area <= 4 pixels at target size
    those segments are dropped and the map is recomputed from the survivors (without the merge).  Segment ids are the
    survivors' positions.  A kept class missing from ``is_thing_map`` raises KeyError.

    CUDA fp32 only (csrc/panoptic.cu): one class launch, then rounds of one label launch over the whole batch with one
    read-back of the areas per round, and one launch writing the int32 target-size maps; the PNG is encoded on the
    host.  ``maps_on_device=True`` adds each image's map as ``"label_map"`` (int32 [H, W] on the model's device), which
    ``PanopticEvaluator.update`` scores without decoding the PNG."""

    def __init__(self, is_thing_map, threshold=0.85, maps_on_device=False):
        super().__init__()
        self.threshold = threshold
        self.is_thing_map = is_thing_map
        self.maps_on_device = maps_on_device

    @torch.no_grad()
    def forward(self, outputs, processed_sizes, target_sizes=None):
        from .panoptic_eval import png_of
        maps, infos = self.label_maps(outputs, processed_sizes, target_sizes)
        host = [m.cpu().numpy() for m in maps]
        preds = []
        for m, d, info in zip(host, maps, infos):
            pred = {"png_string": png_of(m), "segments_info": info}
            if self.maps_on_device:
                pred["label_map"] = d
            preds.append(pred)
        return preds

    @torch.no_grad()
    def label_maps(self, outputs, processed_sizes, target_sizes=None, lib=None):
        """The target-size id maps (int32 [H, W] on the outputs' device) and each image's ``segments_info``: what
        ``forward`` returns before the PNG encode.  ``lib``: a ctypes library with the C entries of csrc/panoptic.cu
        (default: the package's) -- the tests pass a host build of the same routines and CPU tensors."""
        from .panoptic_eval import MAX_KEPT, BLOCK_PIXELS, _library, check, stream_of
        if target_sizes is None:
            target_sizes = processed_sizes
        assert len(processed_sizes) == len(target_sizes)
        logits, masks = outputs["pred_logits"], outputs["pred_masks"]
        assert len(logits) == len(masks) == len(target_sizes)
        if lib is None and not (logits.is_cuda and masks.is_cuda):
            raise NotImplementedError("PostProcessPanoptic runs on CUDA outputs (csrc/panoptic.cu)")
        dev = logits.device
        lib, stream = lib or _library(), stream_of(dev)
        B, Q, C = logits.shape
        h, w = masks.shape[-2:]
        logits = logits.float().contiguous()
        masks = masks.float().reshape(B, Q, h, w).contiguous()
        to_hw = lambda s: tuple(int(v) for v in (s.tolist() if torch.is_tensor(s) else s))
        sizes = [to_hw(s) for s in processed_sizes]
        tsizes = [to_hw(s) for s in target_sizes]

        cls = torch.empty(B * Q, dtype=torch.int32, device=dev)
        score = torch.empty(B * Q, dtype=torch.float32, device=dev)
        keep = torch.empty(B * Q, dtype=torch.uint8, device=dev)
        check(lib.tfb200_panoptic_classes_f32(logits.data_ptr(), B, Q, C, float(self.threshold), cls.data_ptr(),
                                              score.data_ptr(), keep.data_ptr(), stream), "panoptic classes")
        cls_h = cls.view(B, Q).cpu().numpy()
        keep_h = keep.view(B, Q).cpu().numpy().astype(bool)

        kept_q, kept_cls, rep, off = [], [], [], [0]
        for b in range(B):
            q = np.nonzero(keep_h[b])[0]
            if len(q) > MAX_KEPT:
                raise ValueError(f"PostProcessPanoptic: image {b} keeps {len(q)} queries, over the limit of {MAX_KEPT}")
            c = cls_h[b, q]
            first_of = {}
            r = np.arange(len(q), dtype=np.int32)
            for k, lab in enumerate(c.tolist()):
                if not self.is_thing_map[lab]:                   # KeyError for an unknown class, as the reference
                    r[k] = first_of.setdefault(lab, k)
            kept_q.append(q.astype(np.int32))
            kept_cls.append(c)
            rep.append(r)
            off.append(off[-1] + len(q))
        n_kept = off[-1]
        max_k = max((len(q) for q in kept_q), default=0)

        # per-image geometry: Pillow's row / column sources and the processed rows / columns' mapped counts
        idx, img = [], np.zeros((B, 14), np.int64)
        io_ = mo = oo = 0
        for b in range(B):
            (H, W), (Ht, Wt) = sizes[b], tsizes[b]
            rows, cols = pillow_nearest_src(H, Ht), pillow_nearest_src(W, Wt)
            parts = [rows, cols, np.bincount(rows, minlength=H), np.bincount(cols, minlength=W)]
            offs = []
            for a in parts:
                offs.append(io_)
                idx.append(a.astype(np.int32))
                io_ += len(a)
            img[b] = (H, W, Ht, Wt, off[b], len(kept_q[b]), mo, offs[0], offs[1], offs[2], offs[3], oo,
                      int(len(kept_q[b]) > 0), 1)
            mo += H * W
            oo += Ht * Wt
        cat = lambda xs: np.concatenate(xs).astype(np.int32) if xs and sum(map(len, xs)) else np.zeros(1, np.int32)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)
        idx_d = up(cat(idx))
        kq_d, rep_d = up(cat(kept_q)), up(cat(rep))
        label = torch.empty(max(mo, 1), dtype=torch.int32, device=dev)
        area = torch.empty(max(n_kept, 1), dtype=torch.int64, device=dev)
        alive = np.ones(max(n_kept, 1), np.int32)
        blocks = max(1, max((H * W + BLOCK_PIXELS - 1) // BLOCK_PIXELS for H, W in sizes))
        areas = np.zeros(n_kept, np.int64)
        while img[:, 12].any():                                  # rounds over the whole batch
            img_d, alive_d = up(img), up(alive)
            area.zero_()
            check(lib.tfb200_panoptic_label_f32(masks.data_ptr(), B, Q, h, w, img_d.data_ptr(), max_k,
                                                kq_d.data_ptr(), alive_d.data_ptr(), rep_d.data_ptr(),
                                                idx_d.data_ptr(), label.data_ptr(), area.data_ptr(), blocks, stream),
                  "panoptic label")
            got = area[:n_kept].cpu().numpy()                   # the round's one read-back
            for b in range(B):
                if not img[b, 12]:
                    continue
                s = slice(off[b], off[b + 1])
                areas[s] = got[s]
                small = (alive[s] == 1) & (got[s] <= 4)
                img[b, 13] = 0                                   # later passes do not merge stuff duplicates
                if small.any():
                    alive[s][small] = 0
                    img[b, 12] = int(alive[s].any())
                else:
                    img[b, 12] = 0
        pos = np.zeros(max(n_kept, 1), np.int32)
        infos = []
        for b in range(B):
            s = slice(off[b], off[b + 1])
            surv = np.nonzero(alive[s] == 1)[0]
            pos[off[b] + surv] = np.arange(len(surv), dtype=np.int32)
            infos.append([{"id": i, "isthing": self.is_thing_map[int(kept_cls[b][k])],
                           "category_id": int(kept_cls[b][k]), "area": int(areas[off[b] + k])}
                          for i, k in enumerate(surv.tolist())])
        out = torch.empty(max(oo, 1), dtype=torch.int32, device=dev)
        img_d = up(img)
        check(lib.tfb200_panoptic_final_f32(img_d.data_ptr(), B, up(alive).data_ptr(), up(pos).data_ptr(),
                                            idx_d.data_ptr(), label.data_ptr(), out.data_ptr(),
                                            max(1, max((Ht * Wt + BLOCK_PIXELS - 1) // BLOCK_PIXELS
                                                       for Ht, Wt in tsizes)), stream), "panoptic final")
        maps = [out[int(img[b, 11]):int(img[b, 11]) + Ht * Wt].view(Ht, Wt) for b, (Ht, Wt) in enumerate(tsizes)]
        return maps, infos
