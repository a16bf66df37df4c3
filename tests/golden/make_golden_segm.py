#!/usr/bin/env python
"""Segmentation-model golden fixtures recorded FROM THE REFERENCE (build container only).

Runs the reference classes DeformableDETRSegm / DeformableDETRSegmTracking, SetCriterion (with the ``masks`` loss) and
PostProcessSegm from /root/reference/src on CPU, set up exactly as tests/golden/make_golden_model.py does (visdom and
the compiled extension stubbed, the pure-PyTorch MSDeformAttn core, no weight downloads), driven by the shared case
runners of tests/segm_fixtures.py, and stores tests/golden/model_segm_<case>.npz.

ONE PATCH of the reference: ``DETRSegmBase.forward(samples, targets)`` (models/detr_segmentation.py:41) has no
``prev_features`` parameter, although the reference tracker calls its detector with three arguments
(models/tracker.py:306), so reference MOTS tracking with a mask model fails with a TypeError.  The recorder wraps that
forward so a third argument is handed to the next class in the MRO (DETRTrackingBase / DeformableDETR) for the
duration of the call; the reference's own body runs unchanged, and the two-argument call is not touched.
"""
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


def patch_prev_features(seg_module):
    base = seg_module.DETRSegmBase
    original = base.forward

    def forward(self, samples, targets=None, prev_features=None):
        if prev_features is None:
            return original(self, samples, targets)
        mro = type(self).__mro__
        nxt = mro[mro.index(base) + 1]
        inner = nxt.forward

        def with_prev(this, s, t=None, *_):
            return inner(this, s, t, prev_features)
        nxt.forward = with_prev
        try:
            return original(self, samples, targets)
        finally:
            nxt.forward = inner
    base.forward = forward


def main():
    import segm_fixtures as sf
    from make_golden_model import import_reference
    build_model, to_ns = import_reference()
    import trackformer.models.detr_segmentation as seg
    patch_prev_features(seg)

    def load(name):
        return yaml.safe_load(open(os.path.join(REF, "cfgs", name)))

    def build(tracking, multi_frame, **overrides):
        cfg = load("train.yaml")
        cfg.update(load("train_deformable.yaml"))
        if tracking:
            cfg.update(load("train_tracking.yaml"))
            cfg["dataset"] = "mot"
        cfg["device"] = "cpu"
        cfg.update(overrides)
        torch.manual_seed(0)
        model, criterion, _ = build_model(to_ns(cfg))
        return model, criterion

    cases = {
        "det_mini": lambda: sf.run_segm_train_step(build, seg.PostProcessSegm),
        "track_two_frames": lambda: sf.run_segm_two_frames(build),
    }
    only = sys.argv[1:]
    for name, fn in cases.items():
        if only and name not in only:
            continue
        res = fn()
        path = os.path.join(HERE, f"model_segm_{name}.npz")
        np.savez_compressed(path, **{k: np.asarray(v) for k, v in res.items()})
        print(f"segm_{name:18s} -> {os.path.relpath(path)} ({os.path.getsize(path)/1024:.0f} KiB)", flush=True)


if __name__ == "__main__":
    main()
