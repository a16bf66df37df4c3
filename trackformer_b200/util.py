"""Small host-side helpers the hot path needs (mirrors of the reference's util functions).

  NestedTensor / nested_tensor_from_tensor_list   src/trackformer/util/misc.py:309-365
  inverse_sigmoid                                 src/trackformer/util/misc.py:515-519
  box_cxcywh_to_xyxy / generalized_box_iou        src/trackformer/util/box_ops.py:9-61
  sigmoid_focal_loss / accuracy                   src/trackformer/util/misc.py:540-571, 447-461
  world-size helpers                              src/trackformer/util/misc.py:392-418
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import Tensor


class NestedTensor:
    """A padded image batch plus its padding mask (True = padded pixel)."""

    def __init__(self, tensors: Tensor, mask: Optional[Tensor] = None):
        self.tensors = tensors
        self.mask = mask

    def to(self, device) -> "NestedTensor":
        return NestedTensor(self.tensors.to(device), None if self.mask is None else self.mask.to(device))

    def decompose(self):
        return self.tensors, self.mask

    def __repr__(self):
        return str(self.tensors)


def nested_tensor_from_tensor_list(images: Sequence[Tensor]) -> NestedTensor:
    """Zero-pad CHW images to the largest H and W of the batch (no rounding), mask marks padding."""
    if torch.is_tensor(images):                           # a dense [B,C,H,W] batch: nothing to pad
        if images.ndim != 4:
            raise ValueError("not supported")
        b, _, h, w = images.shape
        mask = torch.zeros((b, h, w), dtype=torch.bool, device=images.device)
        mask._no_padding = True                           # known without looking at the data (no host sync)
        mask._no_padding_version = mask._version          # ... for as long as nobody writes into it (backbone.Joiner)
        return NestedTensor(images, mask)
    first = images[0]
    if first.ndim != 3:
        raise ValueError("not supported")
    c = max(int(im.shape[0]) for im in images)
    h = max(int(im.shape[1]) for im in images)
    w = max(int(im.shape[2]) for im in images)
    batch = torch.zeros((len(images), c, h, w), dtype=first.dtype, device=first.device)
    mask = torch.ones((len(images), h, w), dtype=torch.bool, device=first.device)
    for i, im in enumerate(images):
        batch[i, : im.shape[0], : im.shape[1], : im.shape[2]].copy_(im)
        mask[i, : im.shape[1], : im.shape[2]] = False
    return NestedTensor(batch, mask)


def inverse_sigmoid(x: Tensor, eps: float = 1e-5) -> Tensor:
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


class _RefineBoxes(torch.autograd.Function):
    @staticmethod
    def forward(ctx, delta, ref, eps):
        from .ext import load
        out = load().refine_boxes_forward(delta, ref, eps)
        ctx.save_for_backward(out, ref)
        ctx.eps = eps
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        from .ext import load
        out, ref = ctx.saved_tensors
        gd, gr = load().refine_boxes_backward(grad_out, out, ref, bool(ctx.needs_input_grad[1]), ctx.eps)
        return gd, (gr if ctx.needs_input_grad[1] else None), None


def refine_boxes(delta: Tensor, reference: Tensor, eps: float = 1e-5) -> Tensor:
    """``sigmoid(delta + inverse_sigmoid(reference))`` -- the box refinement of the decoder / detection heads
    (models/deformable_transformer.py:412-422, models/deformable_detr.py:229-248).  ``reference`` has 4 components or 2
    (then only ``delta[..., :2]`` gets it added).  One fused launch per direction on CUDA fp32 tensors, the
    reference's op chain otherwise."""
    if delta.is_cuda and delta.dtype == torch.float32 and reference.dtype == torch.float32 and delta.shape[-1] == 4:
        return _RefineBoxes.apply(delta, reference, eps)
    ref = inverse_sigmoid(reference, eps)
    if ref.shape[-1] == 4:
        return (delta + ref).sigmoid()
    return torch.cat([delta[..., :2] + ref, delta[..., 2:]], -1).sigmoid()


# ----------------------------------------------------------------------------- boxes
def box_cxcywh_to_xyxy(b: Tensor) -> Tensor:
    cx, cy, w, h = b.unbind(-1)
    return torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], dim=-1)


def box_xyxy_to_cxcywh(b: Tensor) -> Tensor:
    x0, y0, x1, y1 = b.unbind(-1)
    return torch.stack([(x0 + x1) / 2, (y0 + y1) / 2, x1 - x0, y1 - y0], dim=-1)


def _area(b: Tensor) -> Tensor:
    return (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])


def box_iou(a: Tensor, b: Tensor):
    area_a, area_b = _area(a), _area(b)
    lt = torch.max(a[:, None, :2], b[:, :2])
    rb = torch.min(a[:, None, 2:], b[:, 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    union = area_a[:, None] + area_b - inter
    return inter / union, union


def _check_boxes(b: Tensor) -> None:
    """Degenerate boxes give inf/nan GIoU: the reference asserts (box_ops.py:51-52).  On CUDA the check is
    asynchronous (device-side assert) so it does not stall the host once per call."""
    ok = (b[:, 2:] >= b[:, :2]).all()
    if b.is_cuda:
        torch._assert_async(ok)
    else:
        assert ok


def generalized_box_iou(a: Tensor, b: Tensor) -> Tensor:
    """Pairwise GIoU of xyxy boxes -> [len(a), len(b)]."""
    _check_boxes(a)
    _check_boxes(b)
    iou, union = box_iou(a, b)
    lt = torch.min(a[:, None, :2], b[:, :2])
    rb = torch.max(a[:, None, 2:], b[:, 2:])
    wh = (rb - lt).clamp(min=0)
    hull = wh[..., 0] * wh[..., 1]
    return iou - (hull - union) / hull


def paired_giou(a: Tensor, b: Tensor) -> Tensor:
    """GIoU of box pairs (a[i], b[i]) -- the diagonal of ``generalized_box_iou(a, b)`` without the matrix."""
    _check_boxes(a)
    _check_boxes(b)
    area_a, area_b = _area(a), _area(b)
    wh = (torch.min(a[:, 2:], b[:, 2:]) - torch.max(a[:, :2], b[:, :2])).clamp(min=0)
    inter = wh[:, 0] * wh[:, 1]
    union = area_a + area_b - inter
    hull_wh = (torch.max(a[:, 2:], b[:, 2:]) - torch.min(a[:, :2], b[:, :2])).clamp(min=0)
    hull = hull_wh[:, 0] * hull_wh[:, 1]
    return inter / union - (hull - union) / hull


# ----------------------------------------------------------------------------- losses
def sigmoid_focal_loss(logits: Tensor, targets: Tensor, num_boxes: float, alpha: float = 0.25,
                       gamma: float = 2) -> Tensor:
    p = logits.sigmoid()
    ce = F.binary_cross_entropy_with_logits(logits, targets, reduction="none")
    p_t = p * targets + (1 - p) * (1 - targets)
    loss = ce * ((1 - p_t) ** gamma)
    if alpha >= 0:
        loss = (alpha * targets + (1 - alpha) * (1 - targets)) * loss
    return loss.mean(1).sum() / num_boxes


def dice_loss(logits: Tensor, targets: Tensor, num_boxes: float) -> Tensor:
    """DICE loss of sigmoid(logits) against binary targets, per row, summed and divided by num_boxes (util/misc.py:522-537)."""
    p = logits.sigmoid().flatten(1)
    numerator = 2 * (p * targets).sum(1)
    denominator = p.sum(-1) + targets.sum(-1)
    return (1 - (numerator + 1) / (denominator + 1)).sum() / num_boxes


@torch.no_grad()
def accuracy(output: Tensor, target: Tensor, topk=(1,)) -> List[Tensor]:
    if target.numel() == 0:
        return [torch.zeros([], device=output.device)]
    k = max(topk)
    _, pred = output.topk(k, 1, True, True)
    hit = pred.t().eq(target.view(1, -1).expand_as(pred.t()))
    return [hit[:kk].reshape(-1).float().sum(0) * (100.0 / target.size(0)) for kk in topk]


# ----------------------------------------------------------------------------- distributed
def is_dist_avail_and_initialized() -> bool:
    return dist.is_available() and dist.is_initialized()


def get_world_size() -> int:
    return dist.get_world_size() if is_dist_avail_and_initialized() else 1


def get_rank() -> int:
    return dist.get_rank() if is_dist_avail_and_initialized() else 0
