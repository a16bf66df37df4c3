"""The vanilla-DETR cases of tests/golden/make_golden_detr.py, driven on trackformer_b200 (test infrastructure).

``build`` is the product twin of the recorder's reference build: cfgs/train.yaml (``vanilla_args``), plus
train_tracking.yaml and the 20-class ``mot`` head for the tracking models.  ``run_case(name, device)`` runs the same
shared runner (tests/model_fixtures.py, tests/segm_fixtures.py) the recorder ran for that case.
"""
import json

import numpy as np
import torch

import model_fixtures as mf
import segm_fixtures as sf


def build(tracking, multi_frame, device="cpu", **overrides):
    from trackformer_b200.model_factory import build_model, vanilla_args
    assert not multi_frame
    if tracking:
        overrides.setdefault("dataset", "mot")
    torch.manual_seed(0)
    model, criterion, _ = build_model(vanilla_args(tracking=tracking, device=device, **overrides))
    return model, criterion


def run_case(name, device="cpu"):
    from trackformer_b200.segmentation import PostProcessSegm
    b = lambda tracking, multi_frame, **kw: build(tracking, multi_frame, **kw)          # noqa: E731
    cases = {
        "det_mini": lambda: mf.run_detection(b, [(160, 224)], device),
        "det_padded_batch": lambda: mf.run_detection(b, [(160, 224), (128, 192)], device),
        "det_800x1333": lambda: mf.run_detection(b, [(800, 1333)], device),
        "track_two_frames": lambda: mf.run_two_frame_tracking(b, (160, 224), 12, device),
        "track_800x1333": lambda: mf.run_two_frame_tracking(b, (800, 1333), 100, device),
        "train_step_det": lambda: mf.run_train_step(b, [(160, 224), (160, 224)], 6, device),
        "train_step_tracking": lambda: mf.run_train_step(b, [(128, 160)], 7, device, tracking=True),
        "segm_det_mini": lambda: sf.run_segm_train_step(b, PostProcessSegm, device),
        "segm_track_two_frames": lambda: sf.run_segm_two_frames(b, device),
    }
    return cases[name]()


def check(res, gold, rtol, rel_atol, skip=()):
    """Every recorded key: strings and integer arrays exactly, floats within rtol and rel_atol x the key's scale."""
    for k, g in gold.items():
        if k in skip:
            continue
        r = np.asarray(res[k])
        if g.dtype.kind in "USbiu":
            np.testing.assert_array_equal(r, g, err_msg=k)
        else:
            scale = max(float(np.abs(g).max()), 1e-6) if g.size else 1.0
            np.testing.assert_allclose(r, g, rtol=rtol, atol=rel_atol * scale, err_msg=k)


def state_dict_layout(model):
    return [[k, list(v.shape)] for k, v in model.state_dict().items()]


def recorded_layout(gold, name):
    return json.loads(str(gold[name]))
