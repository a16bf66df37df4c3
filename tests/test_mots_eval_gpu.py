"""MOTS evaluation on the H100: csrc/mots_eval.cu through `evaluate_mots_accums` against the host build of the same
source (bit for bit, sum of d included) and the oracle of tests/mots_eval_reference.py; several sequences of different
frame sizes in one call against each alone; the MOTS20-train-sized fragmented workload; a cross-check with `mot_eval` on
rectangles; and end to end over MultiSequenceTracker(..., mask_rle=True)."""
import numpy as np
import pytest

import mots_eval_fixtures as msf
import mots_eval_reference as ref
from test_mots_eval_cpu import boundary_scenes, check_summary, host_counters, host_lib, oracle_counts, \
    worked_example  # noqa: F401  (host_lib: the module fixture)
from trackformer_b200 import mot_eval, mots, mots_eval

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def _synthetic(seed):
    rng = np.random.default_rng(seed)
    size = [(96, 160), (64, 128), (120, 200), (480, 640)][seed % 4]
    r, g = msf.scene(seed, n_frames=int(rng.integers(5, 30)), n_objects=int(rng.integers(1, 10)), size=size,
                     style="fragmented" if seed % 3 == 2 else "person", p_switch=float(rng.uniform(0, 0.1)))
    return r, g, max([f + 1 for tr in g.values() for f in tr], default=1)


def _evaluate(named, host_lib):
    accums = [mots_eval.get_mots_accum(*v) for v in named.values()]
    out, _ = mots_eval.evaluate_counters(accums, names=list(named))
    host = host_counters(host_lib, accums, list(named))
    assert out.tobytes() == host.tobytes()
    summary, text = mots_eval.evaluate_mots_accums(accums, list(named))
    counts = {n: oracle_counts(*v) for n, v in named.items()}
    check_summary(summary, ref.evaluate(counts))
    for s, c in enumerate(counts.values()):
        assert out[s, 15:16].view(np.float64)[0] == c["sum_d"]
    return accums, out, summary, text


def test_cuda_equals_host_build_and_oracle_and_repeats(dev, host_lib):
    named = {"example": worked_example(), **boundary_scenes(), **{f"seq{s}": _synthetic(s) for s in range(16)}}
    accums, out, summary, text = _evaluate(named, host_lib)
    again, _ = mots_eval.evaluate_counters(accums)
    assert again.tobytes() == out.tobytes()
    assert summary["smotsa"]["example"] == 0.0625


def test_sequences_together_equal_each_alone(dev):
    named = {f"seq{s}": _synthetic(s) for s in range(8)}
    accums = [mots_eval.get_mots_accum(*v) for v in named.values()]
    together, _ = mots_eval.evaluate_counters(accums)
    for s, a in enumerate(accums):
        alone, _ = mots_eval.evaluate_counters([a])
        assert alone.tobytes() == together[s:s + 1].tobytes()


def test_mots20_sized_fragmented_workload_matches_oracle(dev):
    """the MOTS20-train-sized workload with fragmented masks (tests/mots_eval_fixtures.py `mots20_workload`: 2,862
    frames, 26,753 GT masks over 226 tracks, about 100 M intervals) against the dense oracle, its frames spread over a
    process pool"""
    import multiprocessing
    import os
    with multiprocessing.get_context("spawn").Pool(min(32, os.cpu_count() or 1)) as pool:
        named = msf.mots20_workload("fragmented", pool)
        accums = [mots_eval.get_mots_accum(*v) for v in named.values()]
        summary, _ = mots_eval.evaluate_mots_accums(accums, list(named))
        counts = {n: ref.counts(*ref.accumulate(*v, pool=pool)) for n, v in named.items()}
    check_summary(summary, ref.evaluate(counts))
    out, z = mots_eval.evaluate_counters(accums)
    for s, c in enumerate(counts.values()):
        assert out[s, 15:16].view(np.float64)[0] == c["sum_d"]
    assert out[:, 16 + mots_eval._XGTDETS].sum() == 26753 and z["n_gt"] == 226
    assert out[:, 16 + mots_eval._XINTERVALS].sum() > 50_000_000


def _rect_scene(seed, n_frames=25, n=8, h=120, w=200):
    """objects on disjoint integer-pixel rectangles (one column band each), hypotheses too, no ignore regions: as
    masks and as boxes"""
    rng = np.random.default_rng(seed)
    band = w // n
    gt_m, res_m, frames, res_b = {k + 1: {} for k in range(n)}, {}, [], {}   # GT ids in ascending order
    for f in range(n_frames):
        gt_b = {}
        for k in range(n):
            if rng.random() < 0.15:
                continue
            x0 = k * band + int(rng.integers(0, 3)); x1 = x0 + int(rng.integers(8, band - 2))
            y0 = int(rng.integers(0, 40)); y1 = y0 + int(rng.integers(20, 80))
            gt_b[k + 1] = np.asarray([x0, y0, x1, y1], np.float32)
            if rng.random() < 0.85:
                t = k + 100 * (f // 9 if k % 3 == 0 else 0)          # id switches
                dx = int(rng.integers(-2, 3)); dy = int(rng.integers(-6, 7))
                hx0, hx1 = max(k * band, x0 + dx), min((k + 1) * band, x1 + dx + int(rng.integers(-2, 3)))
                hy0, hy1 = max(0, y0 + dy), min(h, y1 + dy + int(rng.integers(-8, 9)))
                if hx1 > hx0 and hy1 > hy0:
                    res_b.setdefault(t, {})[f] = {"bbox": np.asarray([hx0, hy0, hx1, hy1], np.float32)}
        frames.append({"gt": gt_b})
    for f, fr in enumerate(frames):
        for o, b in fr["gt"].items():
            gt_m[o][f] = {"mask": _box_rle(b, h, w), "class_id": 2}
    for t, tr in res_b.items():
        for f, d in tr.items():
            res_m.setdefault(t, {})[f] = {"mask": _box_rle(d["bbox"], h, w)}
    return (res_m, {o: tr for o, tr in gt_m.items() if tr}, n_frames), (res_b, frames)


def _box_rle(b, h, w):
    x0, y0, x1, y1 = (int(v) for v in b)
    return msf.rle([[c * h + y0, c * h + y1] for c in range(x0, x1)], h, w)


def test_rectangles_equal_mot_eval_on_boxes(dev):
    masks, boxes = {}, {}
    for s in range(6):
        m, b = _rect_scene(s)
        masks[f"s{s}"], boxes[f"s{s}"] = m, b
    ms_acc = [mots_eval.get_mots_accum(*v) for v in masks.values()]
    mo_acc = [mot_eval.get_mot_accum(*v) for v in boxes.values()]
    ms, _ = mots_eval.evaluate_mots_accums(ms_acc, list(masks))
    mo, _ = mot_eval.evaluate_mot_accums(mo_acc, list(boxes))
    for col in ("num_unique_objects", "mostly_tracked", "partially_tracked", "mostly_lost", "num_false_positives",
                "num_misses", "num_switches", "num_fragmentations", "idf1", "idp", "idr", "recall", "precision"):
        np.testing.assert_array_equal(ms[col].to_numpy(), mo[col].to_numpy(), err_msg=col)
    np.testing.assert_allclose(ms["motsp"].to_numpy(), 1.0 - mo["motp"].to_numpy(), rtol=0, atol=1e-15)
    c_ms, _ = mots_eval.evaluate_counters(ms_acc)
    c_mo, _ = mot_eval.evaluate_counters(mo_acc)
    assert c_ms[:, :16].tobytes() == c_mo.tobytes()             # every counter, sum of d bit for bit
    assert (ms["num_ignored"] == 0).all()


def _scene_gt(scene, n_frames, size):
    """the scene's objects as disjoint masks: each object's box painted in id order, later ones on top"""
    h, w = size
    gt = {}
    for t in range(n_frames):
        label = np.full((h, w), -1, np.int32)
        for j in range(scene.n):
            if scene.alive(j, t):
                cx, cy, bw, bh = scene.box(j, t)
                x0, x1 = int(max(0, (cx - bw / 2) * w)), int(min(w, (cx + bw / 2) * w))
                y0, y1 = int(max(0, (cy - bh / 2) * h)), int(min(h, (cy + bh / 2) * h))
                label[y0:y1, x0:x1] = j
        for j in range(scene.n):
            if (label == j).any():
                gt.setdefault(j, {})[t] = {"mask": mots.encode(label == j), "class_id": 2}
    return gt


def test_multi_sequence_tracker_end_to_end(dev):
    """the six scripted MOTS cases tracked together (tests/test_multi_tracker_masks_cpu.py's run) scored against their
    scenes' objects in one call; the same run with bool masks gives the identical summary"""
    import tracker_fixtures as tf
    from test_multi_tracker_masks_cpu import _run_cases
    from trackformer_b200 import multi_tracker as mt
    summaries = []
    for mask_rle in (True, False):
        cases, tr, _, _ = _run_cases(None, mask_rle, device=dev, cls=mt.MultiSequenceTracker)
        gt = _scene_gt(tf.Scene(seed=0), tf.N_FRAMES, (tf.IMG_H, tf.IMG_W))
        accums = [mots_eval.get_mots_accum(tr.sequence(s).results, gt, tf.N_FRAMES) for s in range(len(cases))]
        summary, text = mots_eval.evaluate_mots_accums(accums, cases)
        summaries.append(summary)
    print(text)
    assert summaries[0].to_numpy(np.float64).tobytes() == summaries[1].to_numpy(np.float64).tobytes()
    assert (summaries[0]["num_detections"] > 0).all()
