"""Set-prediction loss of the forward+backward hot path.

Mirror of ``SetCriterion`` (src/trackformer/models/detr.py:139-443) for the losses the Deformable-DETR /
TrackFormer configs use -- ``labels`` (sigmoid focal or weighted cross-entropy), ``boxes`` (L1 + GIoU) and
``cardinality`` (logging only) -- applied to the last decoder layer and to every auxiliary layer with its own
Hungarian matching, normalised by the world-averaged number of boxes (one scalar all-reduce, :399-401).
Two-stage models add ``enc_outputs``, the encoder proposals scored against class-agnostic targets (every label 0)
with their own matching (:425-441), under ``_enc`` keys; on CUDA that is one matching-cost launch, the workspace
Hungarian solver (every memory token is a query) and one pass of the fused loss, with no host synchronisation.
``masks`` (sigmoid focal + dice on the bilinearly upsampled mask logits, :330-357) applies to the last layer only;
on CUDA fp32 it is csrc/mask_head.cu, which samples the low-resolution logits at every target pixel on the fly
instead of materialising the upsampled masks.
"""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F
from torch import nn

from .util import (accuracy, box_cxcywh_to_xyxy, dice_loss, generalized_box_iou, get_world_size,
                   is_dist_avail_and_initialized, paired_giou, sigmoid_focal_loss)

_MASK_ALPHA, _MASK_GAMMA = 0.25, 2.0          # loss_masks uses sigmoid_focal_loss's defaults (detr.py:353)


class _MaskLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, src, tgt_masks, tgt, num_boxes):
        from . import ext
        out, stats = ext.load().mask_loss_forward(logits, src, tgt_masks, tgt, num_boxes, _MASK_ALPHA, _MASK_GAMMA)
        ctx.save_for_backward(logits, src, tgt_masks, tgt, stats, num_boxes)
        return out[0], out[1]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_mask, g_dice):
        from . import ext
        logits, src, tgt_masks, tgt, stats, num_boxes = ctx.saved_tensors
        g2 = torch.stack([g_mask, g_dice]).float()
        grad = ext.load().mask_loss_backward(logits, src, tgt_masks, tgt, stats, num_boxes, g2, _MASK_ALPHA, _MASK_GAMMA)
        return grad, None, None, None, None


def _padded_target_masks(targets, device):
    """All target masks of the batch as one [T, Hmax, Wmax] bool tensor, zero-padded to the largest image
    (nested_tensor_from_tensor_list of detr.py:343, indexed by global box number instead of (image, box))."""
    masks = [t["masks"] for t in targets]
    h = max(m.shape[-2] for m in masks)
    w = max(m.shape[-1] for m in masks)
    out = torch.zeros((sum(len(m) for m in masks), h, w), dtype=torch.bool, device=device)
    ofs = 0
    for m in masks:
        out[ofs:ofs + len(m), :m.shape[-2], :m.shape[-1]] = m.to(device=device, dtype=torch.bool)
        ofs += len(m)
    return out


def mask_losses(pred_masks, src, tgt, targets, num_boxes):
    """loss_mask / loss_dice of the matched pairs: row ``src[i]`` of ``pred_masks.flatten(0, 1)`` against global target
    mask ``tgt[i]``.  Padding pixels count, as in the reference; no pairs give zero losses."""
    dev = pred_masks.device
    tmasks = _padded_target_masks(targets, dev)
    src, tgt = src.to(dev), tgt.to(dev)
    logits = pred_masks.flatten(0, 1)
    if pred_masks.is_cuda and pred_masks.dtype == torch.float32:
        nb = num_boxes if torch.is_tensor(num_boxes) else torch.tensor(float(num_boxes))
        nb = nb.to(dev, torch.float32).reshape(1)
        loss_mask, loss_dice = _MaskLoss.apply(logits.contiguous(), src, tmasks, tgt, nb)
        return {"loss_mask": loss_mask, "loss_dice": loss_dice}
    sm = F.interpolate(logits[src][:, None], size=tmasks.shape[-2:], mode="bilinear", align_corners=False)
    sm = sm[:, 0].flatten(1)
    tm = tmasks[tgt].flatten(1).to(sm)
    return {"loss_mask": sigmoid_focal_loss(sm, tm, num_boxes, _MASK_ALPHA, _MASK_GAMMA),
            "loss_dice": dice_loss(sm, tm, num_boxes)}



# SetCriterion losses (+ their backward) as fused device kernels (csrc/set_loss.cu)
_FUSED_LOSS = os.environ.get("TFB200_FUSED_LOSS", "1") != "0"


class _SetLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets, n_gt, num_boxes, alpha, gamma, row_valid=None):
        from . import ext
        if row_valid is None:
            out, ul, u1, ug = ext.load().set_loss_forward(logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets, n_gt,
                                                          num_boxes, alpha, gamma)
        else:                                   # rows outside the mask (filler track queries) count for nothing
            out, ul, u1, ug = ext.load().set_loss_forward_masked(logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets,
                                                                 n_gt, num_boxes, row_valid, alpha, gamma)
        ctx.save_for_backward(ul, u1, ug, num_boxes)
        ce, l1, giou, card, cerr = out.unbind(0)
        ctx.mark_non_differentiable(card, cerr)
        return ce, l1, giou, card, cerr

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_ce, g_l1, g_giou, _g_card, _g_err):
        from . import ext
        ul, u1, ug, num_boxes = ctx.saved_tensors
        gl, gb = ext.load().set_loss_backward(ul, u1, ug, g_ce.contiguous(), g_l1.contiguous(), g_giou.contiguous(),
                                              num_boxes)
        return gl, gb, None, None, None, None, None, None, None, None, None, None


class _SetLossSoftmax(torch.autograd.Function):
    """``_SetLoss`` with the weighted cross-entropy of the softmax classifier: loss_ce[k] is normalised by the layer's
    own weight sum (returned by the forward kernel, read by the backward one); ``row_pin`` (optional) marks the
    false-positive track queries that keep their full weight."""
    @staticmethod
    def forward(ctx, logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets, n_gt, num_boxes, eos_coef, row_valid, row_pin):
        from . import ext
        out, ul, u1, ug = ext.load().set_loss_forward_softmax(logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets, n_gt,
                                                              num_boxes, row_valid, row_pin, eos_coef)
        ctx.save_for_backward(ul, u1, ug, num_boxes, out[5])
        ce, l1, giou, card, cerr = out[:5].unbind(0)
        ctx.mark_non_differentiable(card, cerr)
        return ce, l1, giou, card, cerr

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_ce, g_l1, g_giou, _g_card, _g_err):
        from . import ext
        ul, u1, ug, num_boxes, ce_norm = ctx.saved_tensors
        gl, gb = ext.load().set_loss_backward_softmax(ul, u1, ug, g_ce.contiguous(), g_l1.contiguous(),
                                                      g_giou.contiguous(), num_boxes, ce_norm)
        return gl, gb, None, None, None, None, None, None, None, None, None, None


class LossDict(dict):
    """The loss dictionary of ``SetCriterion.forward_stacked`` (reference keys, detr.py:404-424) that also carries the
    per-layer loss VECTORS ``stacked = (loss_ce [K], loss_bbox [K], loss_giou [K])`` its entries are views of: a
    training step can then form the weighted total with three launches instead of one multiply and one add per
    (loss, layer) entry forward and again backward (~110 single-element launches per step at K = 6).

    ``matched = (bat, src, tgt)`` are the last layer's matched pairs as int64 device tensors, image after image: query
    ``src[i]`` of image ``bat[i]`` against global target ``tgt[i]`` (boxes of all images concatenated);
    ``matched_sizes`` are the host counts of pairs per image.  The mask loss reads only these pairs, so a training step
    can run the mask head on those rows alone."""
    stacked = None
    matched = None
    matched_sizes = None


class SetCriterion(nn.Module):
    def __init__(self, num_classes, matcher, weight_dict, eos_coef, losses, focal_loss, focal_alpha,
                 focal_gamma, tracking, track_query_false_positive_eos_weight):
        super().__init__()
        self.num_classes = num_classes
        self.matcher = matcher
        self.weight_dict = weight_dict
        self.eos_coef = eos_coef
        self.losses = losses
        w = torch.ones(num_classes + 1)
        w[-1] = eos_coef
        self.register_buffer("empty_weight", w)
        self.focal_loss = focal_loss
        self.focal_alpha = focal_alpha
        self.focal_gamma = focal_gamma
        self.tracking = tracking
        self.track_query_false_positive_eos_weight = track_query_false_positive_eos_weight
        # solve the assignment problems on the GPU (csrc/lsa.cu) when the outputs live there; TFB200_DEVICE_LSA=0
        # restores the reference's host scipy path
        self.device_matcher = os.environ.get("TFB200_DEVICE_LSA", "1") != "0"
        self._index_memo = {}

    # ---- index helpers -----------------------------------------------------------------------
    @staticmethod
    def _src_idx(indices):
        batch = torch.cat([torch.full_like(src, i) for i, (src, _) in enumerate(indices)])
        return batch, torch.cat([src for src, _ in indices])

    def _target_classes(self, logits, targets, indices):
        idx = self._src_idx(indices)
        matched = torch.cat([t["labels"][j] for t, (_, j) in zip(targets, indices)])
        classes = torch.full(logits.shape[:2], self.num_classes, dtype=torch.int64, device=logits.device)
        classes[idx] = matched
        return idx, matched, classes

    # ---- losses ------------------------------------------------------------------------------
    def loss_labels(self, outputs, targets, indices, _, log=True):
        logits = outputs["pred_logits"]
        idx, matched, classes = self._target_classes(logits, targets, indices)
        ce = F.cross_entropy(logits.transpose(1, 2), classes, weight=self.empty_weight, reduction="none")
        if self.tracking and self.track_query_false_positive_eos_weight:
            for i, t in enumerate(targets):
                if "track_query_boxes" in t:
                    fp = t["track_queries_fal_pos_mask"]
                    ce[i, fp] *= 1 / self.eos_coef            # false track queries are not down-weighted ...
                    classes = classes.clone()
                    classes[i, fp] = 0                        # ... and count with an object-class weight
        out = {"loss_ce": ce.sum() / self.empty_weight[classes].sum()}
        if log:
            out["class_error"] = 100 - accuracy(logits[idx], matched)[0]
        return out

    def loss_labels_focal(self, outputs, targets, indices, num_boxes, log=True):
        logits = outputs["pred_logits"]
        idx, matched, classes = self._target_classes(logits, targets, indices)
        onehot = torch.zeros([logits.shape[0], logits.shape[1], logits.shape[2] + 1], dtype=logits.dtype,
                             device=logits.device)
        onehot.scatter_(2, classes.unsqueeze(-1), 1)
        loss = sigmoid_focal_loss(logits, onehot[:, :, :-1], num_boxes, alpha=self.focal_alpha,
                                  gamma=self.focal_gamma) * logits.shape[1]
        out = {"loss_ce": loss}
        if log:
            out["class_error"] = 100 - accuracy(logits[idx], matched)[0]
        return out

    @torch.no_grad()
    def loss_cardinality(self, outputs, targets, indices, num_boxes):
        logits = outputs["pred_logits"]
        n_gt = torch.as_tensor([len(t["labels"]) for t in targets], device=logits.device)
        n_pred = (logits.argmax(-1) != logits.shape[-1] - 1).sum(1)
        return {"cardinality_error": F.l1_loss(n_pred.float(), n_gt.float())}

    def loss_boxes(self, outputs, targets, indices, num_boxes):
        idx = self._src_idx(indices)
        src = outputs["pred_boxes"][idx]
        tgt = torch.cat([t["boxes"][i] for t, (_, i) in zip(targets, indices)], dim=0)
        l1 = F.l1_loss(src, tgt, reduction="none")
        giou = 1 - torch.diag(generalized_box_iou(box_cxcywh_to_xyxy(src), box_cxcywh_to_xyxy(tgt)))
        return {"loss_bbox": l1.sum() / num_boxes, "loss_giou": giou.sum() / num_boxes}

    def loss_masks(self, outputs, targets, indices, num_boxes):
        assert "pred_masks" in outputs
        n_q, dev = outputs["pred_masks"].shape[1], outputs["pred_masks"].device
        offsets = [0]
        for t in targets:
            offsets.append(offsets[-1] + len(t["masks"]))
        src = torch.cat([s.to(dev) + b * n_q for b, (s, _) in enumerate(indices)])
        tgt = torch.cat([j.to(dev) + offsets[b] for b, (_, j) in enumerate(indices)])
        return mask_losses(outputs["pred_masks"], src, tgt, targets, num_boxes)

    def get_loss(self, loss, outputs, targets, indices, num_boxes, **kwargs):
        table = {"labels": self.loss_labels_focal if self.focal_loss else self.loss_labels,
                 "cardinality": self.loss_cardinality, "boxes": self.loss_boxes, "masks": self.loss_masks}
        assert loss in table, f"do you really want to compute {loss} loss?"
        return table[loss](outputs, targets, indices, num_boxes, **kwargs)

    def forward(self, outputs, targets, num_boxes=None):
        return self._forward(outputs, targets, num_boxes)[0]

    def _forward(self, outputs, targets, num_boxes=None, masks=True):
        """``forward`` -> (losses, the last layer's indices); ``masks=False`` leaves the mask losses out."""
        last = {k: v for k, v in outputs.items() if k != "aux_outputs"}
        aux_list = list(outputs.get("aux_outputs", ()))
        if hasattr(self.matcher, "match_layers"):
            all_indices = self.matcher.match_layers([last] + aux_list, targets)     # one host sync for all layers
        else:
            all_indices = [self.matcher(o, targets) for o in [last] + aux_list]
        indices = all_indices[0]

        n_boxes = sum(len(t["labels"]) for t in targets)
        if num_boxes is not None:
            pass                                # the caller already ran the (collective) normaliser for this step
        elif is_dist_avail_and_initialized():
            t = torch.as_tensor([n_boxes], dtype=torch.float, device=next(iter(outputs.values())).device)
            torch.distributed.all_reduce(t)
            num_boxes = torch.clamp(t / get_world_size(), min=1).item()
        else:
            num_boxes = float(max(n_boxes, 1))

        losses = {}
        for name in self.losses:
            if name == "masks" and not masks:
                continue
            losses.update(self.get_loss(name, outputs, targets, indices, num_boxes))
        for i, aux in enumerate(aux_list):
            for name in self.losses:
                if name == "masks":
                    continue
                kw = {"log": False} if name == "labels" else {}
                part = self.get_loss(name, aux, targets, all_indices[i + 1], num_boxes, **kw)
                losses.update({f"{k}_{i}": v for k, v in part.items()})
        if "enc_outputs" in outputs:
            losses.update(self._encoder_losses_host(outputs["enc_outputs"], targets, num_boxes))
        return losses, indices

    @staticmethod
    def _binary_targets(targets):
        """the targets with every label 0 (detr.py:427-429; only boxes and labels are read)"""
        return [{"boxes": t["boxes"], "labels": torch.zeros_like(t["labels"])} for t in targets]

    def _encoder_losses_host(self, enc_outputs, targets, num_boxes):
        """the ``_enc`` losses of detr.py:425-441: the matcher and the loss functions on class-agnostic targets"""
        bin_targets = self._binary_targets(targets)
        indices = self.matcher(enc_outputs, bin_targets)
        losses = {}
        for name in self.losses:
            if name == "masks":
                continue
            kw = {"log": False} if name == "labels" else {}
            part = self.get_loss(name, enc_outputs, bin_targets, indices, num_boxes, **kw)
            losses.update({f"{k}_enc": v for k, v in part.items()})
        return losses

    def _encoder_losses(self, enc_logits, enc_boxes, targets, num_boxes):
        """``_encoder_losses_host`` for stacked callers; on CUDA fp32 one ``match_cost`` + ``lsa`` (the workspace solver:
        every token is a query) and one K = 1 pass of the fused loss, nothing read back."""
        bin_targets = self._binary_targets(targets)
        sizes = [len(t["labels"]) for t in targets]
        match = None
        if (self.device_matcher and _FUSED_LOSS and enc_logits.dtype == torch.float32
                and hasattr(self.matcher, "match_layers_device")
                and set(self.losses) - {"masks"} == {"labels", "boxes", "cardinality"}):
            match = self.matcher.match_layers_device(enc_logits.detach()[None], enc_boxes.detach()[None], bin_targets)
        if match is None:
            if num_boxes is None:
                num_boxes = self._num_boxes(targets, enc_logits.device)
            return self._encoder_losses_host({"pred_logits": enc_logits, "pred_boxes": enc_boxes}, targets, num_boxes)
        src2d, tgt2d, status = match
        torch._assert_async(status[0] == 0)
        dev = enc_logits.device
        key = ("n_gt", tuple(sizes), dev)
        n_gt = self._index_memo.get(key)
        if n_gt is None:
            n_gt = self._index_memo[key] = torch.as_tensor(sizes, dtype=torch.float, device=dev)
        if num_boxes is None:
            num_boxes = self._num_boxes(targets, dev)
        fused = self._fused_losses(enc_logits[None], enc_boxes[None], src2d, tgt2d, bin_targets, sizes, n_gt, num_boxes)
        return {f"{k}_enc": fused[k] for k in ("loss_ce", "loss_bbox", "loss_giou", "cardinality_error")}

    @staticmethod
    def _matched_of(indices, targets, device):
        """``LossDict.matched`` / ``matched_sizes`` from per-image host indices [(src, tgt)]"""
        sizes = [len(s) for s, _ in indices]
        ofs, bat, tgt = 0, [], []
        for b, ((_, j), t) in enumerate(zip(indices, targets)):
            bat.append(torch.full((len(j),), b, dtype=torch.int64))
            tgt.append(j.to(torch.int64) + ofs)
            ofs += len(t["labels"])
        src = torch.cat([s.to(torch.int64).cpu() for s, _ in indices])
        idx = torch.stack([torch.cat(bat), src, torch.cat(tgt).cpu()]).to(device, non_blocking=True)
        return (idx[0], idx[1], idx[2]), sizes

    # ------------------------------------------------------------------------------------------
    def _num_boxes(self, targets, device):
        n_boxes = sum(len(t["labels"]) for t in targets)
        if is_dist_avail_and_initialized():
            t = torch.as_tensor([n_boxes], dtype=torch.float, device=device)
            torch.distributed.all_reduce(t)
            return torch.clamp(t / get_world_size(), min=1).item()
        return float(max(n_boxes, 1))

    def num_boxes_device(self, targets, device, out=None):
        """The loss normaliser of detr.py:397-401 as a 0-dim DEVICE tensor: mean box count over the ranks, at least 1,
        without reading anything back (one scalar all-reduce when several ranks run).  ``out`` receives the value in
        place, so a captured step can read it from a static buffer."""
        t = torch.tensor(float(sum(len(t["labels"]) for t in targets)), dtype=torch.float32).to(device, non_blocking=True)
        if is_dist_avail_and_initialized():
            torch.distributed.all_reduce(t)
            t = t / get_world_size()
        t = torch.clamp(t, min=1)
        if out is not None:
            out.copy_(t)
            return out
        return t

    def _false_positive_pins(self, targets, nq, device):
        """``row_pin`` of the matcher when false-positive track queries keep their full class weight (detr.py:190-197:
        ``tracking`` and ``track_query_false_positive_eos_weight``), else None.  A valid row with pin -2 is one."""
        if not (self.tracking and self.track_query_false_positive_eos_weight):
            return None
        return self.matcher.row_pin(targets, nq, device)

    def _fused_losses(self, logits, boxes, src2d, tgt2d, targets, sizes, n_gt, num_boxes, row_valid=None,
                      row_pin=None):
        """The loss values of ``forward_stacked`` and their gradients from three launches (csrc/set_loss.cu)."""
        k = logits.shape[0]
        dev = logits.device
        key = ("off", tuple(sizes), dev)
        off = self._index_memo.get(key)
        if off is None:
            acc = [0]
            for n in sizes:
                acc.append(acc[-1] + n)
            off = self._index_memo[key] = torch.tensor(acc, dtype=torch.int32, device=dev)
        if not torch.is_tensor(num_boxes):
            num_boxes = torch.tensor(float(num_boxes), dtype=torch.float32, device=dev)
        tgt_ids = torch.cat([t["labels"] for t in targets])
        tgt_boxes = torch.cat([t["boxes"] for t in targets]).float()
        if self.focal_loss:
            ce, l1, gi, card, cerr = _SetLoss.apply(logits, boxes, src2d, tgt2d, tgt_ids, tgt_boxes, off, n_gt,
                                                    num_boxes.reshape(1).float(), float(self.focal_alpha),
                                                    float(self.focal_gamma), row_valid)
        else:
            ce, l1, gi, card, cerr = _SetLossSoftmax.apply(logits, boxes, src2d, tgt2d, tgt_ids, tgt_boxes, off, n_gt,
                                                           num_boxes.reshape(1).float(), float(self.eos_coef),
                                                           row_valid, row_pin)
        losses = LossDict({"loss_ce": ce[-1], "class_error": cerr[-1], "loss_bbox": l1[-1], "loss_giou": gi[-1],
                           "cardinality_error": card[-1]})
        for i in range(k - 1):
            losses[f"loss_ce_{i}"] = ce[i]
            losses[f"loss_bbox_{i}"] = l1[i]
            losses[f"loss_giou_{i}"] = gi[i]
            losses[f"cardinality_error_{i}"] = card[i]
        losses.stacked = (ce, l1, gi)
        return losses

    def forward_stacked(self, logits, boxes, targets, num_boxes=None, pred_masks=None, track_queries=False,
                        enc_outputs=None):
        """Same losses as ``forward`` for a detector whose K decoder layers arrive stacked --
        ``logits [K,B,Q,C]``, ``boxes [K,B,Q,4]``, last layer = final prediction -- computed in ONE pass over
        all layers instead of K passes (the reference loops, detr.py:404-424): one Hungarian transfer, one focal
        loss, one L1/GIoU evaluation.  Keys and values equal ``forward`` on the equivalent dict (up to fp32
        summation order); falls back to it for the cases that need per-layer bookkeeping.  With the ``masks`` loss,
        ``pred_masks [B,Q,h,w]`` of the last layer is scored against the last layer's matching; without
        ``pred_masks`` the mask losses are left out, for a caller that scores the masks of ``LossDict.matched`` itself.

        ``track_queries=True`` opts tracking targets (``track_query_match_ids`` ...) into this pass instead of the
        fallback: the track-query forcing of the matcher applies to every layer (on the device when it can, else on
        the host), and ``track_query_padding [Kb]`` (True = filler row, as fed to the decoder) marks rows that are
        neither matched nor scored -- they add nothing to any loss and get no gradient, and the class loss is
        normalised as in the unpadded model.

        Both classifiers take this pass: the sigmoid focal loss (``focal_loss``) and the weighted cross-entropy of the
        softmax classifier, whose false-positive track queries keep their full weight when ``tracking`` and
        ``track_query_false_positive_eos_weight`` are set (detr.py:190-197).

        ``enc_outputs = (logits [B,S,C], boxes [B,S,4])`` of a two-stage model's encoder head adds the ``_enc`` losses of
        ``forward`` (see ``_encoder_losses``)."""
        losses = self._forward_stacked(logits, boxes, targets, num_boxes, pred_masks, track_queries, enc_outputs)
        if enc_outputs is not None and not any(k.endswith("_enc") for k in losses):
            losses.update(self._encoder_losses(enc_outputs[0], enc_outputs[1], targets, num_boxes))
        return losses

    def _forward_stacked(self, logits, boxes, targets, num_boxes, pred_masks, track_queries, enc_outputs):
        k, bs, nq, _ = logits.shape
        layers = [{"pred_logits": logits[i], "pred_boxes": boxes[i]} for i in range(k)]
        with_masks = "masks" in self.losses
        special = (set(self.losses) - {"masks"} != {"labels", "boxes", "cardinality"}
                   or not hasattr(self.matcher, "match_layers"))
        forced = track_queries and any("track_query_match_ids" in t or "track_query_padding" in t for t in targets)
        sizes = [len(t["labels"]) for t in targets]
        if forced and (special or not hasattr(self.matcher, "match_layers_forced")):
            if any("track_query_padding" in t for t in targets):
                raise NotImplementedError("filler track-query rows need the box-only criterion")
            forced = False
        if not forced and (special or any("track_query_match_ids" in t for t in targets)
                           or min(sizes) == 0 or max(sizes) > nq):
            out = dict(layers[-1])
            if with_masks and pred_masks is not None:
                out["pred_masks"] = pred_masks
            out["aux_outputs"] = layers[:-1]
            if enc_outputs is not None:
                out["enc_outputs"] = {"pred_logits": enc_outputs[0], "pred_boxes": enc_outputs[1]}
            if not with_masks:
                return self.forward(out, targets, num_boxes)
            found, indices = self._forward(out, targets, num_boxes, masks=pred_masks is not None)
            losses = LossDict(found)
            losses.matched, losses.matched_sizes = self._matched_of(indices, targets, logits.device)
            return losses

        dev = logits.device
        per_layer = sum(sizes)
        row_valid = None
        if forced and any("track_query_padding" in t for t in targets):
            row_valid = torch.stack([torch.cat([~t["track_query_padding"].to(dev),
                                                torch.ones(nq - len(t["track_query_padding"]), dtype=torch.bool,
                                                           device=dev)])
                                     if "track_query_padding" in t else torch.ones(nq, dtype=torch.bool, device=dev)
                                     for t in targets])                                          # [B, Q]
        device_match = None
        if self.device_matcher and hasattr(self.matcher, "match_layers_device"):
            device_match = self.matcher.match_layers_device(logits.detach(), boxes.detach(), targets, forced=True) \
                if forced else self.matcher.match_layers_device(logits.detach(), boxes.detach(), targets)
        if device_match is not None:
            # Hungarian matching on the device: no host synchronisation anywhere in the loss
            src2d, tgt2d, status = device_match
            torch._assert_async(status[0] == 0)
            key = (tuple(sizes), k, dev)
            memo = self._index_memo.get(key)
            if memo is None:
                lay = torch.arange(k).repeat_interleave(per_layer)
                bat = torch.cat([torch.full((n,), b, dtype=torch.int64) for b, n in enumerate(sizes)]).repeat(k)
                memo = self._index_memo[key] = (lay.to(dev), bat.to(dev),
                                                torch.as_tensor(sizes, dtype=torch.float, device=dev))
            lay, bat, n_gt = memo
            src, tgt = src2d.reshape(-1), tgt2d.reshape(-1)
            if num_boxes is None:               # callers replaying a captured step pass the (static) normaliser in
                num_boxes = self._num_boxes(targets, dev)
        elif forced:
            all_indices = self.matcher.match_layers_forced(logits.detach(), boxes.detach(), targets)
        else:
            all_indices = self.matcher.match_layers(layers, targets)        # [K][B] (src, tgt) on the host
        if device_match is None:
            if num_boxes is None:
                num_boxes = self._num_boxes(targets, dev)
            lay = torch.arange(k).repeat_interleave(per_layer)
            bat = torch.cat([torch.full_like(src, b) for ind in all_indices for b, (src, _) in enumerate(ind)])
            src = torch.cat([s_ for ind in all_indices for (s_, _) in ind])
            tgt = torch.cat([t_ + off for ind in all_indices
                             for (_, t_), off in zip(ind, [sum(sizes[:b]) for b in range(bs)])])
            idx = torch.stack([lay, bat, src, tgt]).to(dev, non_blocking=True)
            lay, bat, src, tgt = idx[0], idx[1], idx[2], idx[3]
            n_gt = torch.as_tensor(sizes, device=dev, dtype=torch.float)
        last = slice((k - 1) * per_layer, None)
        last_pairs = (bat[last], src[last].long(), tgt[last])
        masks = {}
        if with_masks and pred_masks is not None:
            masks = mask_losses(pred_masks, bat[last] * nq + src[last], tgt[last], targets, num_boxes)
        row_pin = self._false_positive_pins(targets, nq, dev) if forced and not self.focal_loss else None
        if device_match is not None and _FUSED_LOSS and logits.dtype == torch.float32:
            losses = self._fused_losses(logits, boxes, src2d, tgt2d, targets, sizes, n_gt, num_boxes,
                                        None if row_valid is None else row_valid.reshape(-1).to(torch.uint8), row_pin)
            losses.update(masks)
            losses.matched, losses.matched_sizes = last_pairs, sizes
            return losses
        gt_labels = torch.cat([t["labels"] for t in targets])[tgt]
        gt_boxes = torch.cat([t["boxes"] for t in targets])[tgt]

        classes = torch.full((k, bs, nq), self.num_classes, dtype=torch.int64, device=dev)
        classes[lay, bat, src] = gt_labels
        if self.focal_loss:
            # labels: sigmoid focal loss against one-hot targets (no-object = all zeros)
            onehot = torch.zeros((k, bs, nq, logits.shape[-1] + 1), dtype=logits.dtype, device=dev)
            onehot.scatter_(3, classes.unsqueeze(-1), 1)
            onehot = onehot[..., :-1]
            p = logits.sigmoid()
            ce = F.binary_cross_entropy_with_logits(logits, onehot, reduction="none")
            p_t = p * onehot + (1 - p) * (1 - onehot)
            focal = ce * ((1 - p_t) ** self.focal_gamma)
            if self.focal_alpha >= 0:
                focal = (self.focal_alpha * onehot + (1 - self.focal_alpha) * (1 - onehot)) * focal
            if row_valid is not None:
                focal = focal * row_valid[None, :, :, None].to(focal.dtype)
            loss_ce = focal.mean(2).sum((1, 2)) / num_boxes * nq                                   # [K]
        else:
            # labels: weighted cross-entropy (detr.py:185-204), each layer normalised by its own weight sum
            weight = self.empty_weight.to(device=dev, dtype=logits.dtype)
            ce = F.cross_entropy(logits.flatten(0, 2), classes.flatten(), weight=weight,
                                 reduction="none").view(k, bs, nq)
            w = weight[classes]
            if row_pin is not None:                      # false-positive track queries: full weight, class-0 normaliser
                fal_pos = row_pin.to(dev).view(bs, nq) == -2
                if row_valid is not None:
                    fal_pos = fal_pos & row_valid
                ce = torch.where(fal_pos, ce * (1 / self.eos_coef), ce)
                w = torch.where(fal_pos, weight[0], w)
            if row_valid is not None:
                ce = ce * row_valid.to(ce.dtype)
                w = w * row_valid.to(w.dtype)
            loss_ce = ce.sum((1, 2)) / w.sum((1, 2))                                                # [K]

        # boxes: L1 + GIoU over the matched pairs of every layer
        matched = boxes[lay, bat, src]
        loss_bbox = (matched - gt_boxes).abs().view(k, per_layer, 4).sum((1, 2)) / num_boxes
        giou = paired_giou(box_cxcywh_to_xyxy(matched), box_cxcywh_to_xyxy(gt_boxes))
        loss_giou = (1 - giou).view(k, per_layer).sum(1) / num_boxes

        with torch.no_grad():
            predicted = logits.argmax(-1) != logits.shape[-1] - 1
            if row_valid is not None:
                predicted = predicted & row_valid[None]
            n_pred = predicted.sum(2).float()                                                    # [K,B]
            card = (n_pred - n_gt[None]).abs().mean(1)                                           # [K]
            last = slice((k - 1) * per_layer, None)
            class_error = 100 - accuracy(logits[-1][bat[last], src[last]], gt_labels[last])[0]

        losses = LossDict({"loss_ce": loss_ce[-1], "class_error": class_error, "loss_bbox": loss_bbox[-1],
                           "loss_giou": loss_giou[-1], "cardinality_error": card[-1]})
        for i in range(k - 1):
            losses[f"loss_ce_{i}"] = loss_ce[i]
            losses[f"loss_bbox_{i}"] = loss_bbox[i]
            losses[f"loss_giou_{i}"] = loss_giou[i]
            losses[f"cardinality_error_{i}"] = card[i]
        losses.stacked = (loss_ce, loss_bbox, loss_giou)
        losses.update(masks)
        losses.matched, losses.matched_sizes = last_pairs, sizes
        return losses
