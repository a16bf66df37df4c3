"""Model factory + the reference's hyper-parameter sets for the hot path.

``build_model(args)`` mirrors src/trackformer/models/__init__.py:16-130 for the deformable, box-only
configurations (detection and tracking): it returns ``(model, criterion, postprocessors)`` with the same class
counts (:17-26), loss weights (:83-99) and focal-loss post-processor (:117-118).

With ``masks=True`` it builds the segmentation models of src/trackformer/models/detr_segmentation.py
(``DeformableDETRSegm`` / ``DeformableDETRSegmTracking``) and adds the ``masks`` loss and the ``segm``
post-processor (:42-45, 86-88, 103-104, 121-125); the panoptic post-processor is not provided.

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
from .deformable_detr import DeformableDETR, DeformablePostProcess
from .deformable_transformer import build_deforamble_transformer
from .detr_tracking import DeformableDETRTracking
from .matcher import build_matcher
from .segmentation import DeformableDETRSegm, DeformableDETRSegmTracking, PostProcessSegm

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


def num_classes_for(dataset: str) -> int:
    if dataset == "coco":
        return 91
    if dataset == "coco_panoptic":
        return 250
    if dataset in ("coco_person", "mot", "mot_crowdhuman", "crowdhuman", "mot_coco_person"):
        return 20
    raise NotImplementedError(dataset)


def build_model(args):
    if not args.deformable:
        raise NotImplementedError("only the deformable path is built (vanilla DETR is outside the hot path)")
    if args.masks and args.dataset == "coco_panoptic":
        raise NotImplementedError("the panoptic post-processor is not provided")
    num_classes = num_classes_for(args.dataset)
    backbone = build_backbone(args)
    matcher = build_matcher(args)
    detr_kwargs = dict(
        backbone=backbone, num_classes=num_classes - 1 if args.focal_loss else num_classes,
        num_queries=args.num_queries, aux_loss=args.aux_loss, overflow_boxes=args.overflow_boxes,
        transformer=build_deforamble_transformer(args), num_feature_levels=args.num_feature_levels,
        with_box_refine=args.with_box_refine, two_stage=args.two_stage,
        multi_frame_attention=args.multi_frame_attention, multi_frame_encoding=args.multi_frame_encoding,
        merge_frame_features=args.merge_frame_features)
    if args.tracking:
        tracking_kwargs = dict(
            track_query_false_positive_prob=args.track_query_false_positive_prob,
            track_query_false_negative_prob=args.track_query_false_negative_prob,
            matcher=matcher, backprop_prev_frame=args.track_backprop_prev_frame)
        if args.masks:
            model = DeformableDETRSegmTracking({"freeze_detr": args.freeze_detr}, tracking_kwargs, detr_kwargs)
        else:
            model = DeformableDETRTracking(tracking_kwargs, detr_kwargs)
    elif args.masks:
        model = DeformableDETRSegm({"freeze_detr": args.freeze_detr}, detr_kwargs)
    else:
        model = DeformableDETR(**detr_kwargs)

    weight_dict = {"loss_ce": args.cls_loss_coef, "loss_bbox": args.bbox_loss_coef, "loss_giou": args.giou_loss_coef}
    if args.masks:
        weight_dict["loss_mask"] = args.mask_loss_coef
        weight_dict["loss_dice"] = args.dice_loss_coef
    if args.aux_loss:
        base = dict(weight_dict)
        for i in range(args.dec_layers - 1):
            weight_dict.update({f"{k}_{i}": v for k, v in base.items()})
    criterion = SetCriterion(
        num_classes, matcher=matcher, weight_dict=weight_dict, eos_coef=args.eos_coef,
        losses=["labels", "boxes", "cardinality"] + (["masks"] if args.masks else []), focal_loss=args.focal_loss, focal_alpha=args.focal_alpha,
        focal_gamma=args.focal_gamma, tracking=args.tracking,
        track_query_false_positive_eos_weight=args.track_query_false_positive_eos_weight)
    criterion.to(torch.device(args.device))
    postprocessors = {"bbox": DeformablePostProcess()}
    if args.masks:
        postprocessors["segm"] = PostProcessSegm()
    return model, criterion, postprocessors
