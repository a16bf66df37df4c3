#!/usr/bin/env python
"""Vanilla-DETR golden fixtures recorded FROM THE REFERENCE (build container only).

Builds the reference's DETR / DETRTracking / DETRSegm / DETRSegmTracking from cfgs/train.yaml (``deformable: false``;
train_tracking.yaml and the 20-class ``mot`` head for the tracking models) on CPU, set up as
tests/golden/make_golden_model.py does, and drives them with the shared case runners of tests/model_fixtures.py and
tests/segm_fixtures.py.  Stores tests/golden/detr_<case>.npz.

ONE SHIM of the reference: ``DETR.forward(samples, targets)`` (models/detr.py:62) and ``DETRSegmBase.forward``
(models/detr_segmentation.py:41) take no ``prev_features``, but ``DETRTrackingBase.forward`` (detr_tracking.py:274) and
the tracker (tracker.py:306) pass one, so the reference's vanilla tracking classes fail with a TypeError.  Both
forwards are wrapped to drop that third argument (vanilla DETR has no multi-frame path); their bodies run unchanged.
"""
import json
import os
import sys

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
REF = "/root/reference"


def drop_prev_features(cls):
    original = cls.forward

    def forward(self, samples, targets=None, prev_features=None):
        return original(self, samples, targets)
    cls.forward = forward


def postprocess_case(post_cls):
    """The reference PostProcess on seeded logits (with exact ties between real classes) and boxes."""
    g = torch.Generator().manual_seed(21)
    logits = torch.randn(2, 50, 21, generator=g) * 3
    logits[0, 3, 5] = logits[0, 3, 2] = logits[0, 3].max() + 1.0          # tie: the smaller class index wins
    boxes = torch.rand(2, 50, 4, generator=g) * 0.5 + 0.1
    sizes = torch.tensor([[480, 640], [750, 1333]])
    res = post_cls()({"pred_logits": logits, "pred_boxes": boxes}, sizes)
    out = {"logits": logits.numpy(), "boxes": boxes.numpy(), "sizes": sizes.numpy()}
    for i, r in enumerate(res):
        for k, v in r.items():
            out[f"{i}/{k}"] = v.numpy()
    return out


def main():
    import model_fixtures as mf
    import segm_fixtures as sf
    from make_golden_model import import_reference
    build_model, to_ns = import_reference()
    import trackformer.models.detr as detr
    import trackformer.models.detr_segmentation as seg
    drop_prev_features(detr.DETR)
    drop_prev_features(seg.DETRSegmBase)

    def load(name):
        return yaml.safe_load(open(os.path.join(REF, "cfgs", name)))

    def build(tracking, multi_frame, **overrides):
        assert not multi_frame
        cfg = load("train.yaml")
        if tracking:
            cfg.update(load("train_tracking.yaml"))
            cfg["dataset"] = "mot"
        cfg["device"] = "cpu"
        cfg.update(overrides)
        torch.manual_seed(0)
        model, criterion, _ = build_model(to_ns(cfg))
        return model, criterion

    def state_dicts():
        res = {}
        for name, tracking, masks in (("DETR", False, False), ("DETRTracking", True, False),
                                      ("DETRSegm", False, True), ("DETRSegmTracking", True, True)):
            model, _ = build(tracking, False, masks=masks)
            assert type(model).__name__ == name
            res[name] = np.asarray(json.dumps([[k, list(v.shape)] for k, v in model.state_dict().items()]))
        return res

    cases = {
        "state_dicts": state_dicts,
        "postprocess": lambda: postprocess_case(detr.PostProcess),
        "det_mini": lambda: mf.run_detection(build, [(160, 224)]),
        "det_padded_batch": lambda: mf.run_detection(build, [(160, 224), (128, 192)]),
        "det_800x1333": lambda: mf.run_detection(build, [(800, 1333)]),
        "track_two_frames": lambda: mf.run_two_frame_tracking(build, (160, 224), 12),
        "track_800x1333": lambda: mf.run_two_frame_tracking(build, (800, 1333), 100),
        "train_step_det": lambda: mf.run_train_step(build, [(160, 224), (160, 224)], 6),
        "train_step_tracking": lambda: mf.run_train_step(build, [(128, 160)], 7, tracking=True),
        "segm_det_mini": lambda: sf.run_segm_train_step(build, seg.PostProcessSegm),
        "segm_track_two_frames": lambda: sf.run_segm_two_frames(build),
    }
    only = sys.argv[1:]
    for name, fn in cases.items():
        if only and name not in only:
            continue
        res = fn()
        path = os.path.join(HERE, f"detr_{name}.npz")
        np.savez(path, **{k: np.asarray(v) for k, v in res.items()})
        print(f"{name:22s} -> {os.path.relpath(path)} ({os.path.getsize(path) / 1024:.0f} KiB)", flush=True)


if __name__ == "__main__":
    main()
