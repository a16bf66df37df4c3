"""Hungarian matcher between predictions and ground-truth boxes.

Mirror of src/trackformer/models/matcher.py:13-141.  The cost matrix (focal / softmax class cost, L1 box
cost, GIoU cost) is built on the GPU; the linear-sum-assignment itself runs on the host with scipy exactly
like the reference (:104,:127) -- the index bookkeeping downstream must stay bit-exact, so the solver is not
swapped.  Track-query forcing (:108-125): false-positive track queries can match nothing, every other track
query is pinned to the ground-truth box of its identity.
"""
from __future__ import annotations

import os

import numpy as np
import torch
from scipy.optimize import linear_sum_assignment
from torch import nn

from .util import box_cxcywh_to_xyxy, generalized_box_iou

# matching cost and SetCriterion losses as fused device kernels (csrc/set_loss.cu)
_FUSED_LOSS = os.environ.get("TFB200_FUSED_LOSS", "1") != "0"


class HungarianMatcher(nn.Module):
    def __init__(self, cost_class: float = 1, cost_bbox: float = 1, cost_giou: float = 1,
                 focal_loss: bool = False, focal_alpha: float = 0.25, focal_gamma: float = 2.0):
        super().__init__()
        assert cost_class != 0 or cost_bbox != 0 or cost_giou != 0, "all costs cant be 0"
        self.cost_class = cost_class
        self.cost_bbox = cost_bbox
        self.cost_giou = cost_giou
        self.focal_loss = focal_loss
        self.focal_alpha = focal_alpha
        self.focal_gamma = focal_gamma
        self._offsets_memo = {}

    def _cost(self, logits, boxes, tgt_ids, tgt_boxes):
        """[Q', C] logits, [Q', 4] boxes against all T ground-truth boxes of the batch -> [Q', T] cost."""
        if self.focal_loss:
            p = logits.sigmoid()
            neg = (1 - self.focal_alpha) * (p ** self.focal_gamma) * (-(1 - p + 1e-8).log())
            pos = self.focal_alpha * ((1 - p) ** self.focal_gamma) * (-(p + 1e-8).log())
            c_class = pos[:, tgt_ids] - neg[:, tgt_ids]
        else:
            c_class = -logits.softmax(-1)[:, tgt_ids]
        c_bbox = torch.cdist(boxes, tgt_boxes, p=1)
        c_giou = -generalized_box_iou(box_cxcywh_to_xyxy(boxes), box_cxcywh_to_xyxy(tgt_boxes))
        return self.cost_bbox * c_bbox + self.cost_class * c_class + self.cost_giou * c_giou

    @torch.no_grad()
    def match_layers(self, outputs_list, targets):
        """Matchings for several decoder layers with ONE device->host transfer (the reference pays one
        ``.cpu()`` sync per layer, detr.py:393,412).  Cost values, and therefore the assignments, are the ones
        ``forward`` computes layer by layer.  Track-query forcing needs per-layer bookkeeping: fall back."""
        if any("track_query_match_ids" in t for t in targets):
            return [self.forward(o, targets) for o in outputs_list]
        bs, nq = outputs_list[0]["pred_logits"].shape[:2]
        tgt_ids = torch.cat([t["labels"] for t in targets])
        tgt_boxes = torch.cat([t["boxes"] for t in targets])
        sizes = [len(t["boxes"]) for t in targets]
        k = len(outputs_list)
        logits = torch.stack([o["pred_logits"] for o in outputs_list]).flatten(0, 2)
        boxes = torch.stack([o["pred_boxes"] for o in outputs_list]).flatten(0, 2)
        cost = self._cost(logits, boxes, tgt_ids, tgt_boxes).view(k, bs, nq, -1).cpu()
        result = []
        for layer in cost:
            picks = [linear_sum_assignment(c[i]) for i, c in enumerate(layer.split(sizes, -1))]
            result.append([(torch.as_tensor(r, dtype=torch.int64), torch.as_tensor(c, dtype=torch.int64))
                           for r, c in picks])
        return result

    @torch.no_grad()
    def match_layers_device(self, logits, boxes, targets):
        """All K layers' matchings ON THE DEVICE (csrc/lsa.cu): no device->host transfer, CUDA-graph capturable.
        ``logits [K,B,Q,C]``, ``boxes [K,B,Q,4]`` -> ``(src [K,T], tgt [K,T], status)`` with T = total number of
        boxes; for image b the columns ``off[b]..off[b+1]-1`` hold its (query, box) pairs in ascending query order --
        the pairs scipy returns (the optimum is unique unless costs tie exactly).  Returns ``None`` when the device
        solver does not apply (track-query forcing, more boxes than queries, CPU tensors)."""
        from . import ext
        k, bs, nq, _ = logits.shape
        sizes = [len(t["boxes"]) for t in targets]
        if (not logits.is_cuda or any("track_query_match_ids" in t for t in targets) or max(sizes) > nq
                or sum(sizes) == 0):
            return None
        tgt_ids = torch.cat([t["labels"] for t in targets])
        tgt_boxes = torch.cat([t["boxes"] for t in targets])
        if _FUSED_LOSS and self.focal_loss and logits.dtype == torch.float32:
            # the whole cost matrix in one launch (csrc/set_loss.cu) instead of ~25 elementwise kernels
            cost = ext.load().match_cost(logits, boxes, tgt_ids, tgt_boxes.float(), self.cost_class, self.cost_bbox,
                                         self.cost_giou, self.focal_alpha, self.focal_gamma).view(k, bs, nq, -1)
        else:
            cost = self._cost(logits.flatten(0, 2), boxes.flatten(0, 2), tgt_ids, tgt_boxes).view(k, bs, nq, -1)
        key = (tuple(sizes), logits.device)
        off = self._offsets_memo.get(key)
        if off is None:
            acc = [0]
            for n in sizes:
                acc.append(acc[-1] + n)
            off = self._offsets_memo[key] = torch.tensor(acc, dtype=torch.int32, device=logits.device)
        return ext.load().lsa(cost.float(), off, max(sizes))

    @torch.no_grad()
    def forward(self, outputs, targets):
        bs, nq = outputs["pred_logits"].shape[:2]
        logits = outputs["pred_logits"].flatten(0, 1)
        boxes = outputs["pred_boxes"].flatten(0, 1)
        tgt_ids = torch.cat([t["labels"] for t in targets])
        tgt_boxes = torch.cat([t["boxes"] for t in targets])
        cost = self._cost(logits, boxes, tgt_ids, tgt_boxes).view(bs, nq, -1).cpu()

        sizes = [len(t["boxes"]) for t in targets]
        for i, t in enumerate(targets):
            if "track_query_match_ids" not in t:
                continue
            col0 = sum(sizes[:i])
            fal_pos = t["track_queries_fal_pos_mask"].tolist()
            is_track = t["track_queries_mask"].tolist()
            match_ids = t["track_query_match_ids"].tolist()
            k = 0
            for j in range(cost.shape[1]):
                if fal_pos[j]:
                    cost[i, j] = np.inf
                elif is_track[j]:
                    col = match_ids[k] + col0
                    k += 1
                    cost[i, j] = np.inf
                    cost[i, :, col] = np.inf
                    cost[i, j, col] = -1
        picks = [linear_sum_assignment(c[i]) for i, c in enumerate(cost.split(sizes, -1))]
        return [(torch.as_tensor(r, dtype=torch.int64), torch.as_tensor(c, dtype=torch.int64)) for r, c in picks]


def build_matcher(args):
    return HungarianMatcher(cost_class=args.set_cost_class, cost_bbox=args.set_cost_bbox,
                            cost_giou=args.set_cost_giou, focal_loss=args.focal_loss,
                            focal_alpha=args.focal_alpha, focal_gamma=args.focal_gamma)
