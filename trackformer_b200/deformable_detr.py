"""Deformable-DETR detector shell around the H100 transformer.

Mirror of ``DETR`` (constructor state only: src/trackformer/models/detr.py:17-54), ``MLP`` (:493-507) and
``DeformableDETR`` (src/trackformer/models/deformable_detr.py:29-283) with the same forward signature
``(samples, targets=None, prev_features=None) -> (out, targets, features_all, memory_per_level, hs)`` and the
same parameter names (``input_proj.{l}.{0,1}``, ``class_embed.{k}``, ``bbox_embed.{k}.layers.{j}``,
``query_embed``, ``transformer.*``, ``backbone.*``).  Two-stage and mask heads are outside the hot path.
"""
from __future__ import annotations

import copy
import math

import torch
import torch.nn.functional as F
from torch import nn

from .backbone import _resize_mask
from .util import (NestedTensor, box_cxcywh_to_xyxy, refine_boxes,
                   nested_tensor_from_tensor_list)


def _clones(module, n):
    return nn.ModuleList([copy.deepcopy(module) for _ in range(n)])


from .fused_linear import linear as fused_linear  # noqa: E402


class MLP(nn.Module):
    """ReLU perceptron: ``num_layers`` Linear layers named ``layers.{i}``."""

    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        dims = [input_dim] + [hidden_dim] * (num_layers - 1) + [output_dim]
        self.layers = nn.ModuleList(nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:]))

    def forward(self, x):
        for i, layer in enumerate(self.layers):
            x = fused_linear(x, layer.weight, layer.bias)
            if i + 1 < self.num_layers:
                x = F.relu(x)
        return x


class DETR(nn.Module):
    """State shared by all DETR variants: heads, query embedding, backbone handle (detr.py:20-54)."""

    def __init__(self, backbone, transformer, num_classes, num_queries, aux_loss=False, overflow_boxes=False):
        super().__init__()
        self.num_queries = num_queries
        self.transformer = transformer
        self.overflow_boxes = overflow_boxes
        self.class_embed = nn.Linear(self.hidden_dim, num_classes + 1)
        self.bbox_embed = MLP(self.hidden_dim, self.hidden_dim, 4, 3)
        self.query_embed = nn.Embedding(num_queries, self.hidden_dim)
        self.input_proj = nn.Conv2d(backbone.num_channels[-1], self.hidden_dim, kernel_size=1)
        self.backbone = backbone
        self.aux_loss = aux_loss

    @property
    def hidden_dim(self):
        return self.transformer.d_model

    @property
    def fpn_channels(self):
        return self.backbone.num_channels[:3][::-1]

    @torch.jit.unused
    def _set_aux_loss(self, outputs_class, outputs_coord):
        return [{"pred_logits": a, "pred_boxes": b} for a, b in zip(outputs_class[:-1], outputs_coord[:-1])]


class _CallScratch:
    """Holder for tensors of the latest forward call (they carry autograd history): kept out of copies and pickles of
    the module, which must stay deep-copyable after a training forward."""
    __slots__ = ("value",)

    def __init__(self):
        self.value = None

    def __deepcopy__(self, memo):
        return _CallScratch()

    def __reduce__(self):
        return (_CallScratch, ())


class DeformableDETR(DETR):
    def __init__(self, backbone, transformer, num_classes, num_queries, num_feature_levels, aux_loss=True,
                 with_box_refine=False, two_stage=False, overflow_boxes=False, multi_frame_attention=False,
                 multi_frame_encoding=False, merge_frame_features=False):
        super().__init__(backbone, transformer, num_classes, num_queries, aux_loss)
        if two_stage:
            raise NotImplementedError("two-stage Deformable-DETR is outside the hot path")
        self.merge_frame_features = merge_frame_features
        self.multi_frame_attention = multi_frame_attention
        self.multi_frame_encoding = multi_frame_encoding
        self.overflow_boxes = overflow_boxes
        self.num_feature_levels = num_feature_levels
        self.query_embed = nn.Embedding(num_queries, self.hidden_dim * 2)    # (positional | content) halves

        chans = backbone.num_channels[-3:]
        if num_feature_levels > 1:
            n_backbone = len(backbone.strides) - 1                             # layer2, layer3, layer4
            proj = []
            for i in range(n_backbone):
                in_ch = chans[i]
                proj.append(nn.Sequential(nn.Conv2d(in_ch, self.hidden_dim, kernel_size=1),
                                          nn.GroupNorm(32, self.hidden_dim)))
            for _ in range(num_feature_levels - n_backbone):                   # extra stride-2 level(s)
                proj.append(nn.Sequential(nn.Conv2d(in_ch, self.hidden_dim, kernel_size=3, stride=2, padding=1),
                                          nn.GroupNorm(32, self.hidden_dim)))
                in_ch = self.hidden_dim
            self.input_proj = nn.ModuleList(proj)
        else:
            self.input_proj = nn.ModuleList([nn.Sequential(
                nn.Conv2d(chans[0], self.hidden_dim, kernel_size=1), nn.GroupNorm(32, self.hidden_dim))])
        self.with_box_refine = with_box_refine
        self.two_stage = two_stage

        prior = 0.01
        self.class_embed.bias.data = torch.ones_like(self.class_embed.bias) * (-math.log((1 - prior) / prior))
        nn.init.zeros_(self.bbox_embed.layers[-1].weight)
        nn.init.zeros_(self.bbox_embed.layers[-1].bias)
        for p in self.input_proj:
            nn.init.xavier_uniform_(p[0].weight, gain=1)
            nn.init.zeros_(p[0].bias)

        n_pred = transformer.decoder.num_layers
        if with_box_refine:
            self.class_embed = _clones(self.class_embed, n_pred)
            self.bbox_embed = _clones(self.bbox_embed, n_pred)
            nn.init.constant_(self.bbox_embed[0].layers[-1].bias.data[2:], -2.0)
            self.transformer.decoder.bbox_embed = self.bbox_embed           # shared with the decoder (refinement)
        else:
            nn.init.constant_(self.bbox_embed.layers[-1].bias.data[2:], -2.0)
            self.class_embed = nn.ModuleList([self.class_embed for _ in range(n_pred)])
            self.bbox_embed = nn.ModuleList([self.bbox_embed for _ in range(n_pred)])
            self.transformer.decoder.bbox_embed = None
        if self.merge_frame_features:
            self.merge_features = _clones(nn.Conv2d(self.hidden_dim * 2, self.hidden_dim, kernel_size=1),
                                          num_feature_levels)

    # ------------------------------------------------------------------------------------------
    def _project_levels(self, frame, frame_feat, prev_features, pos, src_list, mask_list, pos_list):
        use_3d = self.multi_frame_attention and self.multi_frame_encoding
        pos_list.extend([p[:, frame] for p in pos[-3:]] if use_3d else pos[-3:])
        for l, feat in enumerate(frame_feat):
            src, mask = feat.decompose()
            assert mask is not None
            if self.merge_frame_features:
                prev_src, _ = prev_features[l].decompose()
                src_list.append(self.merge_features[l](
                    torch.cat([self.input_proj[l](src), self.input_proj[l](prev_src)], dim=1)))
            else:
                src_list.append(self.input_proj[l](src))
            mask_list.append(mask)
        n_have = len(frame_feat)
        for l in range(n_have, self.num_feature_levels):                      # coarser levels made from layer4
            if l == n_have:
                if self.merge_frame_features:
                    src = self.merge_features[l](torch.cat(
                        [self.input_proj[l](frame_feat[-1].tensors), self.input_proj[l](prev_features[-1].tensors)],
                        dim=1))
                else:
                    src = self.input_proj[l](frame_feat[-1].tensors)
            else:
                src = self.input_proj[l](src_list[-1])
            mask = _resize_mask(frame_feat[0].mask, src.shape[-2:])
            pos_l = self.backbone[1](NestedTensor(src, mask)).to(src.dtype)
            src_list.append(src)
            mask_list.append(mask)
            pos_list.append(pos_l[:, frame] if use_3d else pos_l)

    def _call_scratch(self) -> _CallScratch:
        holder = self.__dict__.get("_scratch")
        if holder is None:
            holder = self.__dict__["_scratch"] = _CallScratch()
        return holder

    @property
    def stacked_heads(self):
        """(logits [layers, N, Q, classes], boxes [layers, N, Q, 4]) of the latest forward call, or None"""
        return self._call_scratch().value

    def forward(self, samples: NestedTensor, targets: list = None, prev_features=None):
        self._call_scratch().value = None                # do not keep the previous call's graph alive
        if not isinstance(samples, NestedTensor):
            samples = nested_tensor_from_tensor_list(samples)
        features_all, pos = self.backbone(samples)
        features = features_all[-3:]
        prev_features = features if prev_features is None else prev_features[-3:]

        src_list, mask_list, pos_list = [], [], []
        frames = [prev_features, features] if self.multi_frame_attention else [features]
        for frame, frame_feat in enumerate(frames):
            self._project_levels(frame, frame_feat, prev_features, pos, src_list, mask_list, pos_list)

        hs, memory, init_reference, inter_references, refined_boxes, _ = self.transformer(
            src_list, mask_list, pos_list, self.query_embed.weight, targets)

        logits = torch.stack([self.class_embed[lvl](hs[lvl]) for lvl in range(hs.shape[0])])
        if refined_boxes is not None and self.with_box_refine and refined_boxes.shape[0] == hs.shape[0]:
            # iterative refinement: the decoder already evaluated bbox_embed[lvl](hs[lvl]) + inverse_sigmoid(reference
            # of layer lvl) -- the reference computes the identical expression again here (deformable_detr.py:229-248)
            boxes = refined_boxes
        else:
            boxes = torch.stack([refine_boxes(self.bbox_embed[lvl](hs[lvl]),
                                              init_reference if lvl == 0 else inter_references[lvl - 1])
                                 for lvl in range(hs.shape[0])])
        # per-layer heads as two tensors [layers, N, Q, .]; the training step takes them from here instead of
        # re-stacking the per-layer slices of the output dictionary (whose backward is a zero-fill + copy per slice)
        self._call_scratch().value = (logits, boxes)

        out = {"pred_logits": logits[-1], "pred_boxes": boxes[-1], "hs_embed": hs[-1]}
        if self.aux_loss:
            out["aux_outputs"] = self._set_aux_loss(logits, boxes)

        # encoder memory re-sliced to one NCHW map per level (consumed by the tracker / mask heads)
        bsz, _, ch = memory.shape
        per_level, ofs = [], 0
        for src in src_list:
            h, w = src.shape[-2:]
            per_level.append(memory[:, ofs:ofs + h * w].permute(0, 2, 1).view(bsz, ch, h, w))
            ofs += h * w
        return out, targets, features_all, per_level, hs


class DeformablePostProcess(nn.Module):
    """Sigmoid scores, best class per query, boxes scaled to the target sizes (deformable_detr.py:286-334).

    On CUDA the whole chain is one launch of the fused kernel (csrc/track_post.cu); `packed()` exposes its
    [N, Q, 6] rows {score, label, x0, y0, x1, y1} so the tracker needs a single device->host copy per frame."""

    @torch.no_grad()
    def packed(self, outputs, target_sizes):
        logits, boxes = outputs["pred_logits"], outputs["pred_boxes"]
        assert len(logits) == len(target_sizes) and target_sizes.shape[1] == 2
        if logits.is_cuda and logits.dtype == torch.float32:
            from .ext import load
            rows, labels = load().detect_postprocess(logits, boxes, target_sizes.to(logits.device, torch.int64))
            rows._labels = labels
            return rows
        scores, labels = logits.sigmoid().max(-1)
        img_h, img_w = target_sizes.unbind(1)
        xyxy = box_cxcywh_to_xyxy(boxes) * torch.stack([img_w, img_h, img_w, img_h], dim=1)[:, None, :]
        rows = torch.cat([scores[..., None], labels[..., None].to(scores.dtype), xyxy.to(scores.dtype)], -1)
        rows._labels = labels
        return rows

    @torch.no_grad()
    def forward(self, outputs, target_sizes, results_mask=None):
        rows = self.packed(outputs, target_sizes)
        results = [{"scores": r[:, 0], "scores_no_object": 1 - r[:, 0], "labels": l, "boxes": r[:, 2:6]}
                   for r, l in zip(rows, rows._labels)]
        if results_mask is not None:
            for i, keep in enumerate(results_mask):
                results[i] = {k: v[keep] for k, v in results[i].items()}
        return results
