"""TrackFormer tracking wrapper: track-query bookkeeping around the Deformable-DETR forward.

Mirror of src/trackformer/models/detr_tracking.py:15-290 -- same class layout
(``DETRTrackingBase`` mixed into ``DeformableDETR``), same mode switches (``train`` / ``tracking``), same
forward signature, and -- because the index bookkeeping has to stay BIT-EXACT -- the same sequence of draws
from the CPU torch generator in ``add_track_queries_to_targets``:

  1. randint(0, min_matched+1)                       how many previous-frame matches survive   (:46)
  2. randint(ceil(fp_prob * kept) + 1)               how many false positives to inject        (:51)
  per sample:
  3. randperm(len(prev matches))[:kept]              false-negative sub-sampling               (:63)
  4. randperm(kept)[:n_fp]                           which survivors spawn a false positive    (:104)
  5. multinomial(weights, 1) | randperm(n_unmatched)[0]   which unmatched query becomes it     (:137,:139)

tests/test_model_parity_cpu.py::test_add_track_queries_bit_exact_against_reference (and the tracking train-step tests on
CPU and GPU) check the resulting index tensors bit-for-bit against fixtures produced by the reference class.  The reference's distance weight uses the x-offset twice (:131) -- kept, since it
changes which index the multinomial draws.
"""
from __future__ import annotations

import math
from contextlib import nullcontext

import torch
from torch import nn

from .deformable_detr import DETR, DeformableDETR
from .matcher import HungarianMatcher
from .util import NestedTensor


class DETRTrackingBase(nn.Module):
    def __init__(self, track_query_false_positive_prob: float = 0.0,
                 track_query_false_negative_prob: float = 0.0, matcher: HungarianMatcher = None,
                 backprop_prev_frame=False):
        # NB: like the reference this runs AFTER the detector's __init__ and must not call nn.Module.__init__
        self._matcher = matcher
        self._track_query_false_positive_prob = track_query_false_positive_prob
        self._track_query_false_negative_prob = track_query_false_negative_prob
        self._backprop_prev_frame = backprop_prev_frame
        self._tracking = False

    def train(self, mode: bool = True):
        self._tracking = False
        return super().train(mode)

    def tracking(self):
        """Inference-time tracking mode: eval() and no target rewriting in forward."""
        self.eval()
        self._tracking = True

    # ------------------------------------------------------------------------------------------
    def add_track_queries_to_targets(self, targets, prev_indices, prev_out, add_false_pos=True):
        """Host-side bookkeeping with ONE device->host transfer (SURVEY 8(f4)).

        The reference interleaves the index logic with device reads: a ``.tolist()`` per sample, a ``weights.cpu()`` per
        injected false positive, ``nonzero`` on device tensors (detr_tracking.py:39-217) -- a dozen synchronisations per
        training step.  Here the previous frame's boxes (and the few identity vectors, if they live on the device) come to
        the host once, every decision is taken there with the same arithmetic (fp32 subtract / square / add / sqrt are
        exactly rounded on both sides) and the same five draws from the CPU generator in the same order, and the results
        go back as index tensors: the embeddings / boxes are gathered on the device with one index each."""
        device = prev_out["pred_boxes"].device
        n_queries_prev = prev_out["pred_boxes"].shape[1]
        boxes_host = prev_out["pred_boxes"].detach().to("cpu")                   # the one device->host transfer

        fewest = min(len(tgt_i) for _, tgt_i in prev_indices)
        n_keep = torch.randint(0, fewest + 1, (1,)).item() if fewest else 0                            # draw 1
        n_fp = 0
        if n_keep:
            n_fp = torch.randint(int(math.ceil(self._track_query_false_positive_prob * n_keep)) + 1, (1,)).item()  # draw 2

        for i, (target, (out_i, tgt_i)) in enumerate(zip(targets, prev_indices)):
            out_i, tgt_i = out_i.to("cpu"), tgt_i.to("cpu")
            if self._track_query_false_negative_prob:
                keep = torch.randperm(len(tgt_i))[:n_keep]                                             # draw 3
                out_i, tgt_i = out_i[keep], tgt_i[keep]

            # identities seen in the previous frame that are still present in the current one
            prev_ids = target["prev_target"]["track_ids"].to("cpu")[tgt_i]
            same_id = prev_ids.unsqueeze(1).eq(target["track_ids"].to("cpu"))
            still_there = same_id.any(dim=1)
            match_ids = same_id.nonzero()[:, 1]

            if add_false_pos:
                matched_xy = boxes_host[i, out_i[still_there]][:, :2]
                taken = set(out_i.tolist())
                free = [q for q in range(n_queries_prev) if q not in taken]
                free_xy = boxes_host[i, :, :2]
                injected = []
                for j in torch.randperm(n_keep)[:n_fp]:                                                # draw 4
                    if len(matched_xy) > j:
                        dx = matched_xy[j].unsqueeze(0) - free_xy[free]
                        weights = torch.sqrt(dx[:, 0] ** 2 + dx[:, 0] ** 2)                            # (sic) x twice
                        pick = torch.multinomial(weights, 1).item()                                    # draw 5a
                    else:
                        pick = torch.randperm(len(free))[0]                                            # draw 5b
                    injected.append(free.pop(pick))
                out_i = torch.tensor(out_i.tolist() + injected).long()
                still_there = torch.cat([still_there, torch.zeros(len(injected), dtype=torch.bool)])

            pad = torch.zeros(self.num_queries, dtype=torch.bool)
            rows = out_i.to(device)
            target["track_query_match_ids"] = match_ids.to(device)
            target["track_query_hs_embeds"] = prev_out["hs_embed"][i].index_select(0, rows)
            target["track_query_boxes"] = prev_out["pred_boxes"][i].index_select(0, rows).detach()
            target["track_queries_mask"] = torch.cat([torch.ones_like(still_there), pad]).to(device)
            target["track_queries_fal_pos_mask"] = torch.cat([~still_there, pad]).to(device)

    # ------------------------------------------------------------------------------------------
    def forward(self, samples: NestedTensor, targets: list = None, prev_features=None, prev_valid=None):
        if targets is not None and not self._tracking:
            prev_targets = [t["prev_target"] for t in targets]
            if self.training:
                ctx = nullcontext if self._backprop_prev_frame else torch.no_grad
                with ctx():
                    if "prev_prev_image" in targets[0]:
                        for t, pt in zip(targets, prev_targets):
                            pt["prev_target"] = t["prev_prev_target"]
                        pp_targets = [t["prev_prev_target"] for t in targets]
                        pp_out, _, pp_features, _, _ = super().forward([t["prev_prev_image"] for t in targets])
                        pp_indices = self._matcher({k: v for k, v in pp_out.items() if "aux_outputs" not in k},
                                                   pp_targets)
                        self.add_track_queries_to_targets(prev_targets, pp_indices, pp_out, add_false_pos=False)
                        prev_out, _, prev_features, _, _ = super().forward(
                            [t["prev_image"] for t in targets], prev_targets, pp_features)
                    else:
                        prev_out, _, prev_features, _, _ = super().forward([t["prev_image"] for t in targets])
                    prev_indices = self._matcher({k: v for k, v in prev_out.items() if "aux_outputs" not in k},
                                                 prev_targets)
                    self.add_track_queries_to_targets(targets, prev_indices, prev_out)
            else:
                # evaluation of plain detection: no track queries
                for t in targets:
                    dev = t["boxes"].device
                    t["track_query_hs_embeds"] = torch.zeros(0, self.hidden_dim).float().to(dev)
                    t["track_queries_mask"] = torch.zeros(self.num_queries).bool().to(dev)
                    t["track_queries_fal_pos_mask"] = torch.zeros(self.num_queries).bool().to(dev)
                    t["track_query_boxes"] = torch.zeros(0, 4).to(dev)
                    t["track_query_match_ids"] = torch.tensor([]).long().to(dev)
        return super().forward(samples, targets, prev_features, prev_valid)


TWO_STAGE_TRACKING = ("two-stage Deformable DETR does not take track queries: its decoder queries are the selected "
                      "encoder proposals, and the reference's two-stage branch skips the track-query concatenation")


class DeformableDETRTracking(DETRTrackingBase, DeformableDETR):
    def __init__(self, tracking_kwargs, detr_kwargs):
        if detr_kwargs.get("two_stage"):
            raise NotImplementedError(TWO_STAGE_TRACKING)
        DeformableDETR.__init__(self, **detr_kwargs)
        DETRTrackingBase.__init__(self, **tracking_kwargs)


class DETRTracking(DETRTrackingBase, DETR):
    def __init__(self, tracking_kwargs, detr_kwargs):
        DETR.__init__(self, **detr_kwargs)
        DETRTrackingBase.__init__(self, **tracking_kwargs)
