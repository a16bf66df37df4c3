"""Tracking with segmentation masks (MOTS) on CPU: trackformer_b200.tracker.Tracker against label maps recorded from
the reference Tracker + PostProcessSegm (tests/golden/make_golden_track_masks.py), the row-selective mask head, word 7
of the device routine's result rows, and the argument checks of the mask-resolution entry point."""
import ctypes
import os

import numpy as np
import pytest
import torch

import track_mask_fixtures as tmf
import tracker_fixtures as tf
from test_track_step_cpu import host_tracker  # noqa: F401  (the g++ build of the device routine, as a fixture)
from test_tracker_cpu import check_against_gold
from trackformer_b200.deformable_detr import DeformablePostProcess
from trackformer_b200.segmentation import PostProcessSegm, resolve_track_masks
from trackformer_b200.tracker import Tracker

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


def check_masks_against_gold(out, name, excused=None):
    """Summary as check_against_gold, then the label maps: equal, except where `excused(frame)` allows a pixel."""
    gold = np.load(os.path.join(GOLD, f"{name}.npz"))
    np.testing.assert_array_equal(out["rows"][:, :3], gold["rows"][:, :3])
    diff = out["labels"] != gold["labels"]
    if excused is None:
        assert not diff.any(), f"{name}: {int(diff.sum())} pixels differ, frames {np.nonzero(diff.any((1, 2)))[0]}"
    else:
        bad = diff & ~excused(gold)
        assert not bad.any(), f"{name}: {int(bad.sum())} unexcused pixels differ"
    return gold


@pytest.mark.parametrize("case", list(tf.CASES))
def test_tracker_masks_match_reference(case):
    out = tmf.run_case(Tracker, DeformablePostProcess(), PostProcessSegm(), case)
    check_against_gold({k: v for k, v in out.items() if k != "labels"}, case)    # masks change no decision
    gold = np.load(os.path.join(GOLD, f"tracker_masks_{case}.npz"))
    for key in gold.files:
        if key != "labels":
            np.testing.assert_array_equal(out[key], gold[key], err_msg=key)
    check_masks_against_gold(out, f"tracker_masks_{case}")


def test_mask_fixtures_exercise_ties_and_stale_masks():
    """the scripted scene must hold saturated overlaps (exact ties) and tracks that keep last frame's mask"""
    scene = tf.Scene()
    det = tmf.MaskedScriptedDetector(scene)
    ties = []

    class Log(torch.nn.Module):
        num_queries, overflow_boxes = det.num_queries, det.overflow_boxes

        def forward(self, *args):
            res = det(*args)
            ties.append(int(((torch.sigmoid(res[0]["pred_masks"][0]) == 1.0).sum(0) >= 2).sum()))
            return res
    tr = Tracker(Log(), {"bbox": DeformablePostProcess(), "segm": PostProcessSegm()}, tf.tracker_cfg("reid_embedding"),
                 False)
    tr.obj_detector.p = torch.nn.Parameter(torch.zeros(1))
    n_stale = 0
    for blob in tmf.blobs(scene):
        tr.step(blob)
        n_stale += int((tr._result_rows < 0).sum())
    assert n_stale > 0 and sum(ties) > 0


def test_masked_detector_keeps_the_scripted_outputs():
    """the masked detector adds pred_masks and changes nothing else; the blobs only gain the "size" entry"""
    scene = tf.Scene()
    a, b = tf.ScriptedDetector(scene), tmf.MaskedScriptedDetector(scene)
    targets = None
    for _ in range(3):
        oa, ob = a(None, targets)[0], b(None, targets)[0]
        assert set(ob) == set(oa) | {"pred_masks"}
        assert ob["pred_masks"].shape == (1, oa["pred_logits"].shape[1]) + tmf.MASK_HW
        for k in oa:
            assert torch.equal(oa[k], ob[k]), k
        targets = [{"track_query_boxes": oa["pred_boxes"][0, -5:], "track_query_hs_embeds": oa["hs_embed"][0, -5:]}]
    for plain, masked in zip(tf.blobs(scene, 2), tmf.blobs(scene, 2)):
        assert set(masked) == set(plain) | {"size"}


def test_resolution_ties_and_stale_masks_by_hand():
    """first maximum wins; stale masks compete with exactly 1.0; > 0.5 only"""
    logits = torch.full((3, 4, 4), -20.0)
    logits[0, :, :2] = 30.0                 # saturated: ties with row 1 and with stale track 7
    logits[1, :, 1:] = 40.0
    logits[2] = 0.0                         # sigmoid 0.5: never foreground
    prev = torch.full((4, 4), -1, dtype=torch.int32)
    prev[2:, :] = 7
    lab = resolve_track_masks(logits, [2, 1, -1, 0], [5, 3, 7, 9], prev, (4, 4), (4, 4), (4, 4))
    want = torch.tensor([[9, 3, 3, 3], [9, 3, 3, 3], [7, 3, 3, 3], [7, 3, 3, 3]], dtype=torch.int32)
    want[2:, 0] = 7                         # stale (position 2) beats row 0 (position 3); row 1 (position 1) beats both
    want[2:, 1:] = 3
    assert torch.equal(lab, want), lab


@pytest.mark.parametrize("seed", range(30))
def test_result_word7_on_random_scenes(host_tracker, seed):
    from test_track_step_cpu import _RandomDetector
    rng = np.random.RandomState(seed)
    cfg = dict(tf.BASE_CFG)
    cfg.update(
        public_detections=[False, "center_distance", "min_iou_0_5"][seed % 3],
        detection_obj_score_thresh=float(rng.uniform(0.5, 0.8)), track_obj_score_thresh=float(rng.uniform(0.4, 0.7)),
        reid_score_thresh=float(rng.uniform(0.4, 0.8)), detection_nms_thresh=float(rng.choice([0.0, 0.3, 0.6])),
        track_nms_thresh=float(rng.choice([0.0, 0.4, 0.7])), steps_termination=int(rng.randint(1, 3)),
        inactive_patience=int(rng.randint(1, 6)), reid_greedy_matching=bool(seed % 2),
        reid_sim_threshold=float(rng.choice([0.0, 3.0, 6.0])), reid_sim_only=seed % 5 == 4)
    trackers, seen = [], [[], []]
    for i, cls in enumerate((Tracker, host_tracker)):
        det = _RandomDetector(seed)
        tr = cls(det, {"bbox": DeformablePostProcess()}, cfg, False)

        class Blob(dict):
            def __getitem__(self, key):
                return det.public if key == "dets" else dict.__getitem__(self, key)
        for t in range(14):
            tr.step(Blob(img=torch.zeros(1, 3, 8, 8), orig_size=torch.tensor([[480, 640]]), dets=None))
            seen[i].append(tr._result_rows.copy())
        trackers.append(tr)
    assert sum(len(r) for r in seen[0]) > 0 and any((r < 0).any() for r in seen[0]) == any((r < 0).any() for r in seen[1])
    for a, b in zip(*seen):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("case", ["reid_embedding", "default"])
def test_device_routine_masks_match_reference(host_tracker, case):
    """DeviceTracker's algorithm (host build) + word 7 + the torch resolution: the reference's label maps"""
    out = tmf.run_case(host_tracker, DeformablePostProcess(), PostProcessSegm(), case)
    check_masks_against_gold(out, f"tracker_masks_{case}")


def test_orig_size_change_with_stale_masks_raises():
    scene = tf.Scene()
    det = tmf.MaskedScriptedDetector(scene)
    tr = Tracker(det, {"bbox": DeformablePostProcess(), "segm": PostProcessSegm()}, tf.tracker_cfg("reid_embedding"),
                 False)
    blobs = list(tmf.blobs(scene))
    raised = False
    for t, blob in enumerate(blobs):
        blob["orig_size"] = torch.tensor([[tf.IMG_H + t, tf.IMG_W]])
        try:
            tr.step(blob)
        except ValueError as e:
            assert "orig_size" in str(e)
            raised = True
            break
    assert raised


def _segm_build():
    from test_model_parity_cpu import build
    return build


@pytest.mark.parametrize("k,bucket", [(0, 8), (5, 8), (8, 8), (11, 4)])
def test_row_selective_head_equals_full_head(k, bucket, monkeypatch):
    """GraphedDetector(use_graphs=False).mask_logits(rows) == the full forward's pred_masks rows, across paddings"""
    from oracle.torch_ref import msda_core_torch
    import model_fixtures as mf
    import trackformer_b200.msda_module as mm
    from trackformer_b200.graphed_detector import GraphedDetector

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    monkeypatch.setattr(mm, "MSDeformAttnFunction", _OracleFn)
    model, _ = _segm_build()(True, False, masks=True)
    mf.canonical_weights_(model, 0)
    model.tracking()
    f1, f2 = tf.model_frames((64, 96), 2)
    with torch.no_grad():
        o1, _, feat1, _, _ = model(f1[None])
        tgt = None
        if k:
            tgt = [{"track_query_boxes": o1["pred_boxes"][0, :k].clone(),
                    "track_query_hs_embeds": o1["hs_embed"][0, :k].clone(), "image_id": torch.tensor([1])}]
        full, *_ = model(f2[None], tgt, feat1)
        det = GraphedDetector(model, bucket=bucket, use_graphs=False)
        out, *_ = det.detect(f2[None], tgt, feat1)
        assert "pred_masks" not in out
        rows = [0, k + 3, k + model.num_queries - 1] + ([k - 1, 1] if k > 1 else [])
        got = det.mask_logits(rows)
    want = full["pred_masks"][:, rows]
    assert got.shape == want.shape
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)
    with torch.no_grad():                                   # the model's own row-selective call
        d_out, _, feats, mem, hs = model.detect(f2[None], tgt, feat1)
        sel = model.mask_logits(feats, mem, hs, rows)
    torch.testing.assert_close(sel, want, rtol=1e-4, atol=1e-4)


def test_track_masks_entry_point_rejects_bad_arguments():
    """-1 NULL pointer, -2 bad shape, 0 for T == 0 (argument checks run before anything touches the device)"""
    from trackformer_b200 import ext
    ext.load()
    lib = ctypes.CDLL(ext.library_path())
    f = lib.tfb200_track_masks_f32
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_int] * 9 + [ctypes.c_void_p]
    buf = (ctypes.c_int32 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ok = (8, 8, 30, 30, 30, 30, 60, 60)
    assert f(None, None, None, None, None, 1, *ok, None) == -1
    assert f(p, p, None, None, p, 1, *ok, None) == -1
    assert f(p, p, p, None, None, 1, *ok, None) == -1
    assert f(p, p, p, None, p, -1, *ok, None) == -2
    assert f(p, p, p, None, p, 1, 0, 8, 30, 30, 30, 30, 60, 60, None) == -2         # h
    assert f(p, p, p, None, p, 1, 8, 8, 30, 30, 31, 30, 60, 60, None) == -2         # crop beyond size
    assert f(p, p, p, None, p, 1, 8, 8, 30, 30, 30, 30, 0, 60, None) == -2          # H
    assert f(p, p, p, None, p, 0, *ok, None) == 0

