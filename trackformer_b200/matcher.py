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
        return self._assign(cost, sizes)

    @staticmethod
    def _assign(cost, sizes):
        """scipy on every (layer, image) block of a host ``cost [K,B,Q,T]`` -> [K][B] (src, tgt)"""
        result = []
        for layer in cost:
            picks = [linear_sum_assignment(c[i]) for i, c in enumerate(layer.split(sizes, -1))]
            result.append([(torch.as_tensor(r, dtype=torch.int64), torch.as_tensor(c, dtype=torch.int64))
                           for r, c in picks])
        return result

    @staticmethod
    def row_pin(targets, num_rows, device):
        """The track-query forcing of ``forward`` (:112-128) as one int32 code per (image, query row), ``[B * num_rows]``:
        -1 free row, -2 excluded row (false-positive track query, or a filler row), c >= 0 row pinned to GLOBAL box
        column c.  The k-th track row that is not a false positive takes ``track_query_match_ids[k]``, as in ``forward``.
        ``track_query_padding [Kb]`` (bool, True = filler) lays the unpadded rows of the masks, in order, onto the
        non-filler rows of a ``[Kb + object queries]`` layout.  Built on the device without reading anything back."""
        pins, col0 = [], 0
        for t in targets:
            pad = t.get("track_query_padding")
            if "track_query_match_ids" in t:
                fal_pos = t["track_queries_fal_pos_mask"].to(device)
                pinned = t["track_queries_mask"].to(device) & ~fal_pos
                ids = t["track_query_match_ids"].to(device=device, dtype=torch.int64)
                ids = torch.cat([ids, ids.new_zeros(1)])                 # keeps the gather defined when there are none
                rank = (pinned.long().cumsum(0) - 1).clamp(min=0)
                pin = torch.where(pinned, ids[rank] + col0, torch.full_like(rank, -1))
                pin = torch.where(fal_pos, torch.full_like(pin, -2), pin)
            else:
                pin = torch.full((num_rows,), -1, dtype=torch.int64, device=device)      # (only the head is read)
            if pad is not None:
                real = torch.cat([~pad.to(device), torch.ones(num_rows - pad.shape[0], dtype=torch.bool, device=device)])
                where = (real.long().cumsum(0) - 1).clamp(min=0)
                pin = torch.where(real, pin[where], torch.full_like(where, -2))
            pins.append(pin)
            col0 += len(t["boxes"])
        return torch.stack(pins).to(torch.int32).reshape(-1)

    @staticmethod
    def force_cost(cost, row_pin):
        """``cost [..., B, Q, T]`` rewritten by ``row_pin [B*Q]`` (see ``row_pin``): the rewrite ``forward`` applies
        (:112-128), in torch.  The device kernel (csrc/set_loss.cu, match_cost_track) applies the same one."""
        bs, nq, n_cols = cost.shape[-3:]
        pin = row_pin.to(cost.device, torch.int64).view(bs, nq)
        pinned = (pin >= 0) & (pin < n_cols)
        excluded = ~pinned & (pin != -1)
        cols = torch.arange(n_cols, device=cost.device)
        col_pinned = torch.zeros(bs, n_cols + 1, dtype=torch.bool, device=cost.device)
        col_pinned.scatter_(1, torch.where(pinned, pin, n_cols), True)
        col_pinned = col_pinned[:, :n_cols]
        inf = torch.full((), float("inf"), dtype=cost.dtype, device=cost.device)
        at_pin = torch.where(cols == pin[..., None], torch.full((), -1.0, dtype=cost.dtype, device=cost.device), inf)
        blocked = excluded[..., None] | col_pinned[:, None, :]
        return torch.where(pinned[..., None], at_pin, torch.where(blocked, inf, cost))

    @torch.no_grad()
    def match_layers_forced(self, logits, boxes, targets):
        """Host route of the forced matching for stacked ``logits [K,B,Q,C]`` / ``boxes [K,B,Q,4]``: the rewrite of
        ``row_pin`` / ``force_cost`` and scipy per layer and image -> [K][B] (src, tgt).  Unlike ``forward`` it accepts
        filler rows (``track_query_padding``); on the real rows it gives ``forward``'s pairs."""
        k, bs, nq, _ = logits.shape
        sizes = [len(t["boxes"]) for t in targets]
        if sum(sizes) == 0:
            empty = torch.zeros(0, dtype=torch.int64)
            return [[(empty, empty) for _ in range(bs)] for _ in range(k)]
        tgt_ids = torch.cat([t["labels"] for t in targets])
        tgt_boxes = torch.cat([t["boxes"] for t in targets])
        cost = self._cost(logits.flatten(0, 2), boxes.flatten(0, 2), tgt_ids, tgt_boxes).view(k, bs, nq, -1)
        cost = self.force_cost(cost, self.row_pin(targets, nq, logits.device)).cpu()
        return self._assign(cost, sizes)

    @torch.no_grad()
    def match_layers_device(self, logits, boxes, targets, forced=False):
        """All K layers' matchings ON THE DEVICE (csrc/lsa.cu): no device->host transfer, CUDA-graph capturable.
        ``logits [K,B,Q,C]``, ``boxes [K,B,Q,4]`` -> ``(src [K,T], tgt [K,T], status)`` with T = total number of
        boxes; for image b the columns ``off[b]..off[b+1]-1`` hold its (query, box) pairs in ascending query order --
        the pairs scipy returns (the optimum is unique unless costs tie exactly).  Returns ``None`` when the device
        solver does not apply (more boxes than queries, no boxes at all, CPU tensors) and, unless ``forced``, for
        targets with track-query forcing.  With ``forced`` the track-query rewrite of ``forward`` (see ``row_pin``,
        filler rows included) is applied to the cost of every layer in the same launch; an image without boxes then
        takes the host route (``match_layers_forced``)."""
        from . import ext
        k, bs, nq, _ = logits.shape
        sizes = [len(t["boxes"]) for t in targets]
        if (not logits.is_cuda or (not forced and any("track_query_match_ids" in t for t in targets))
                or max(sizes) > nq or sum(sizes) == 0 or (forced and min(sizes) == 0)):
            return None
        tgt_ids = torch.cat([t["labels"] for t in targets])
        tgt_boxes = torch.cat([t["boxes"] for t in targets])
        fused = _FUSED_LOSS and logits.dtype == torch.float32
        # focal: (alpha, gamma) after the weights; softmax: the weights alone
        cls_args = (self.focal_alpha, self.focal_gamma) if self.focal_loss else ()
        if forced:
            pin = self.row_pin(targets, nq, logits.device)
            if fused:
                fn = ext.load().match_cost_track if self.focal_loss else ext.load().match_cost_track_softmax
                cost = fn(logits, boxes, tgt_ids, tgt_boxes.float(), pin, self.cost_class, self.cost_bbox,
                          self.cost_giou, *cls_args)
            else:
                cost = self._cost(logits.flatten(0, 2), boxes.flatten(0, 2), tgt_ids, tgt_boxes).view(k, bs, nq, -1)
                cost = self.force_cost(cost, pin)
        elif fused:
            # the whole cost matrix in one launch (csrc/set_loss.cu) instead of ~25 elementwise kernels
            fn = ext.load().match_cost if self.focal_loss else ext.load().match_cost_softmax
            cost = fn(logits, boxes, tgt_ids, tgt_boxes.float(), self.cost_class, self.cost_bbox, self.cost_giou,
                      *cls_args).view(k, bs, nq, -1)
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
