"""Model factory + the reference's hyper-parameter sets for the hot path.

``build_model(args)`` mirrors src/trackformer/models/__init__.py:16-130: it returns ``(model, criterion,
postprocessors)`` with the same class counts (:17-26), model classes (:48-83: ``DeformableDETR[Tracking]`` or, with
``deformable=False``, the vanilla ``DETR[Tracking]``), loss weights (:83-99) and post-processor (:120-123: sigmoid
``DeformablePostProcess`` with the focal loss, softmax ``PostProcess`` otherwise).

With ``masks=True`` it builds the segmentation models of src/trackformer/models/detr_segmentation.py
(``[Deformable]DETRSegm`` / ``[Deformable]DETRSegmTracking``) and adds the ``masks`` loss and the ``segm``
post-processor (:42-45, 86-88, 103-104, 121-125); with ``dataset="coco_panoptic"`` (250 classes, softmax head only) also
the ``panoptic`` post-processor (:124-128).

With ``two_stage=True`` (deformable, ``with_box_refine`` required) it builds two-stage Deformable DETR and adds the
``_enc`` loss weights of the encoder proposals (:99-100).

``vanilla_args(...)`` gives cfgs/train.yaml alone (vanilla DETR), optionally with train_tracking.yaml.
``default_args(...)`` reproduces the values of cfgs/train.yaml overlaid with train_deformable.yaml and,
optionally, train_tracking.yaml / train_multi_frame.yaml (the named sacred configs of src/train.py:24-35), so
the benchmark and the tests can instantiate the exact reference geometry without the YAML files (they do not
exist on the GPU box).  These are data (hyper-parameters), not code.
"""
from __future__ import annotations

from argparse import Namespace

import torch

from .backbone import build_backbone
from .criterion import SetCriterion
from .deformable_detr import DETR, DeformableDETR, DeformablePostProcess, PostProcess
from .deformable_transformer import build_deforamble_transformer
from .detr_tracking import DeformableDETRTracking, DETRTracking
from .matcher import build_matcher
from .segmentation import (PANOPTIC_SIGMOID, DeformableDETRSegm, DeformableDETRSegmTracking, DETRSegm, DETRSegmTracking,
                           PostProcessPanoptic, PostProcessSegm)
from .transformer import build_transformer

_TRAIN_YAML = dict(   # cfgs/train.yaml (model / loss keys only)
    lr=2e-4, lr_backbone_names=["backbone.0"], lr_backbone=2e-5,
    lr_linear_proj_names=["reference_points", "sampling_offsets"], lr_linear_proj_mult=0.1, lr_track=1e-4,
    batch_size=2, weight_decay=1e-4, clip_max_norm=0.1,
    deformable=False, with_box_refine=False, two_stage=False, freeze_detr=False,
    backbone="resnet50", dilation=False, position_embedding="sine", num_feature_levels=1,
    enc_layers=6, dec_layers=6, dim_feedforward=2048, hidden_dim=256, dropout=0.1, nheads=8, num_queries=100,
    pre_norm=False, dec_n_points=4, enc_n_points=4,
    tracking=False, track_prev_frame_range=0, track_prev_prev_frame=False, track_backprop_prev_frame=False,
    track_query_false_positive_prob=0.1, track_query_false_negative_prob=0.4,
    track_query_false_positive_eos_weight=True, track_attention=False,
    multi_frame_attention=False, multi_frame_encoding=True, multi_frame_attention_separate_encoder=True,
    merge_frame_features=False, overflow_boxes=False, masks=False,
    set_cost_class=1.0, set_cost_bbox=5.0, set_cost_giou=2.0,
    aux_loss=True, mask_loss_coef=1.0, dice_loss_coef=1.0, cls_loss_coef=1.0, bbox_loss_coef=5.0, giou_loss_coef=2,
    eos_coef=0.1, focal_loss=False, focal_alpha=0.25, focal_gamma=2,
    dataset="coco", device="cuda", seed=42,
)
_DEFORMABLE_YAML = dict(   # cfgs/train_deformable.yaml
    deformable=True, num_feature_levels=4, num_queries=300, dim_feedforward=1024, focal_loss=True,
    focal_alpha=0.25, focal_gamma=2, cls_loss_coef=2.0, set_cost_class=2.0, overflow_boxes=True,
    with_box_refine=True,
)
_TRACKING_YAML = dict(tracking=True, track_prev_frame_range=5, track_query_false_positive_eos_weight=True)
_MULTI_FRAME_YAML = dict(num_queries=500, hidden_dim=288, multi_frame_attention=True, multi_frame_encoding=True,
                         multi_frame_attention_separate_encoder=True)


def default_args(tracking: bool = False, multi_frame: bool = False, **overrides) -> Namespace:
    cfg = dict(_TRAIN_YAML)
    cfg.update(_DEFORMABLE_YAML)
    if tracking:
        cfg.update(_TRACKING_YAML)
        cfg["dataset"] = "mot"          # 20-class head (models/__init__.py:21-23)
    if multi_frame:
        cfg.update(_MULTI_FRAME_YAML)
    cfg.update(overrides)
    return Namespace(**cfg)


def vanilla_args(tracking: bool = False, masks: bool = False, **overrides) -> Namespace:
    """cfgs/train.yaml as it stands (vanilla DETR: ``deformable: false``, 100 queries, softmax classifier) and, with
    ``tracking``, train_tracking.yaml on top; ``masks`` sets the segmentation head."""
    cfg = dict(_TRAIN_YAML)
    if tracking:
        cfg.update(_TRACKING_YAML)
    cfg["masks"] = masks
    cfg.update(overrides)
    return Namespace(**cfg)


def num_classes_for(dataset: str) -> int:
    if dataset == "coco":
        return 91
    if dataset == "coco_panoptic":
        return 250
    if dataset in ("coco_person", "mot", "mot_crowdhuman", "crowdhuman", "mot_coco_person"):
        return 20
    raise NotImplementedError(dataset)


def build_model(args):
    if args.masks and args.dataset == "coco_panoptic" and args.focal_loss:
        raise NotImplementedError(PANOPTIC_SIGMOID)
    if args.two_stage and not (args.deformable and args.with_box_refine):
        raise ValueError("two_stage needs the deformable model with with_box_refine: its decoder refines the selected "
                         "encoder proposals with the per-layer box heads")
    num_classes = num_classes_for(args.dataset)
    backbone = build_backbone(args)
    matcher = build_matcher(args)
    detr_kwargs = dict(
        backbone=backbone, num_classes=num_classes - 1 if args.focal_loss else num_classes,
        num_queries=args.num_queries, aux_loss=args.aux_loss, overflow_boxes=args.overflow_boxes)
    tracking_kwargs = dict(
        track_query_false_positive_prob=args.track_query_false_positive_prob,
        track_query_false_negative_prob=args.track_query_false_negative_prob,
        matcher=matcher, backprop_prev_frame=args.track_backprop_prev_frame)
    mask_kwargs = {"freeze_detr": args.freeze_detr}
    if args.deformable:
        detr_kwargs.update(
            transformer=build_deforamble_transformer(args), num_feature_levels=args.num_feature_levels,
            with_box_refine=args.with_box_refine, two_stage=args.two_stage,
            multi_frame_attention=args.multi_frame_attention, multi_frame_encoding=args.multi_frame_encoding,
            merge_frame_features=args.merge_frame_features)
        classes = (DeformableDETR, DeformableDETRTracking, DeformableDETRSegm, DeformableDETRSegmTracking)
    else:
        detr_kwargs["transformer"] = build_transformer(args)
        classes = (DETR, DETRTracking, DETRSegm, DETRSegmTracking)
    plain, tracking, segm, segm_tracking = classes
    if args.tracking:
        if args.masks:
            model = segm_tracking(mask_kwargs, tracking_kwargs, detr_kwargs)
        else:
            model = tracking(tracking_kwargs, detr_kwargs)
    elif args.masks:
        model = segm(mask_kwargs, detr_kwargs)
    else:
        model = plain(**detr_kwargs)

    weight_dict = {"loss_ce": args.cls_loss_coef, "loss_bbox": args.bbox_loss_coef, "loss_giou": args.giou_loss_coef}
    if args.masks:
        weight_dict["loss_mask"] = args.mask_loss_coef
        weight_dict["loss_dice"] = args.dice_loss_coef
    if args.aux_loss:
        base = dict(weight_dict)
        for i in range(args.dec_layers - 1):
            weight_dict.update({f"{k}_{i}": v for k, v in base.items()})
        if args.two_stage:
            weight_dict.update({f"{k}_enc": v for k, v in base.items()})
    criterion = SetCriterion(
        num_classes, matcher=matcher, weight_dict=weight_dict, eos_coef=args.eos_coef,
        losses=["labels", "boxes", "cardinality"] + (["masks"] if args.masks else []), focal_loss=args.focal_loss, focal_alpha=args.focal_alpha,
        focal_gamma=args.focal_gamma, tracking=args.tracking,
        track_query_false_positive_eos_weight=args.track_query_false_positive_eos_weight)
    criterion.to(torch.device(args.device))
    postprocessors = {"bbox": DeformablePostProcess() if args.focal_loss else PostProcess()}
    if args.masks:
        postprocessors["segm"] = PostProcessSegm()
        if args.dataset == "coco_panoptic":
            is_thing_map = {i: i <= 90 for i in range(201)}
            postprocessors["panoptic"] = PostProcessPanoptic(is_thing_map, threshold=0.85)
    return model, criterion, postprocessors
