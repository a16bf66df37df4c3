"""MOT evaluation on the H100: csrc/mot_eval.cu through `evaluate_mot_accums` against the oracle of
tests/mot_eval_reference.py -- integer metrics exactly, ratios within 1e-12, per sequence and OVERALL -- on the seeded
synthetic scenes, at MOT20 density, at the stated component limits (and one step above them: a raised error from the
returned status), and end to end over `track_sequences` with the scripted detectors of tests/multi_tracker_fixtures.py.
"""
import time

import numpy as np
import pytest
import torch

import mot_eval_fixtures as mf
import mot_eval_reference as ref
from test_mot_eval_cpu import check_hand_scenes, check_summary, hand_scenes, oracle_counts
from trackformer_b200 import mot_eval

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def _evaluate(named):
    accums = [mot_eval.get_mot_accum(r, fr) for r, fr in named.values()]
    summary, text = mot_eval.evaluate_mot_accums(accums, list(named))
    check_summary(summary, ref.evaluate({n: oracle_counts(r, fr) for n, (r, fr) in named.items()}))
    return accums, summary, text


def _synthetic(seed):
    rng = np.random.default_rng(1000 + seed)
    kw = dict(n_frames=int(rng.integers(20, 60)), n_objects=int(rng.integers(3, 25)),
              p_swap=float(rng.uniform(0, 0.05)), p_dup=float(rng.uniform(0, 0.2)), fp_rate=float(rng.uniform(0, 2)))
    if seed % 3 == 2:
        kw.update(width=120.0, height=160.0, n_objects=int(rng.integers(8, 30)))
    return mf.scene(seed, **kw)


def test_synthetic_scenes_match_oracle_and_repeat_bit_for_bit(dev):
    named = {f"seq{s}": _synthetic(s) for s in range(30)}
    accums, summary, text = _evaluate(named)
    again, text2 = mot_eval.evaluate_mot_accums(accums, list(named))
    assert text == text2
    a, b = summary.to_numpy(np.float64), again.to_numpy(np.float64)
    assert a.tobytes() == b.tobytes()
    c1, _ = mot_eval.evaluate_counters(accums)
    c2, _ = mot_eval.evaluate_counters(accums)
    assert c1.tobytes() == c2.tobytes()


def test_hand_scenes(dev):
    _, summary, _ = _evaluate(hand_scenes())
    check_hand_scenes(summary)


def test_crowded_frames_over_256_objects(dev):
    """about 600 objects per frame (more than one per thread of the CTA) in clumps of 2-6: multi-box residual
    components in most frames"""
    named = {f"clumps{s}": mf.clumps(10 + s) for s in range(3)}
    accums, _, _ = _evaluate(named)
    assert min(int(np.diff(a.frame_obj).min()) for a in accums) > 512
    out, _ = mot_eval.evaluate_counters(accums)
    assert out[:, 11].max() >= 4 and out[:, 12].max() >= 4


def test_mot20_density(dev):
    """three sequences of 2,000 frames with ~150 people per frame in a 1920 x 1080 image"""
    named = {f"MOT20-{s:02d}": mf.scene(50 + s, n_frames=2000, n_objects=150, size=(45.0, 110.0), fp_rate=3.0,
                                          p_swap=0.0005, p_restart=0.002)
             for s in range(3)}
    accums, summary, _ = _evaluate(named)
    out, _ = mot_eval.evaluate_counters(accums)
    print(f"valid pairs {out[:, 1].sum()}, largest residual component {out[:, 11].max()} x {out[:, 12].max()}, "
          f"largest identity component {out[:, 13].max()} x {out[:, 14].max()}")
    assert sum(len(a.obj_id) for a in accums) > 3 * 2000 * 100


def _grid_boxes(n, cell=40.0, cols=40):
    """n boxes far enough apart that no two of them overlap"""
    i = np.arange(n)
    x, y = (i % cols) * cell * 2, (i // cols) * cell * 2
    return np.stack([x, y, x + cell, y + cell], 1)


def _clump(n, rng):
    """n near-identical boxes: every pair of them valid, continuous jitter against ties"""
    base = np.array([100.0, 100.0, 200.0, 300.0])
    return (base + rng.uniform(0, 1.0, (n, 4))).astype(np.float32)


@pytest.mark.parametrize("side", [mot_eval.MAX_CLEAR_COMPONENT, mot_eval.MAX_CLEAR_COMPONENT + 1])
def test_clear_component_limit(dev, side):
    rng = np.random.default_rng(side)
    gt, hy = _clump(side, rng), _clump(side, rng)
    frames = [{"gt": {k + 1: gt[k] for k in range(side)}}, {"gt": {k + 1: gt[k] + 0.5 for k in range(side)}}]
    results = {100 + k: {0: {"bbox": hy[k]}, 1: {"bbox": hy[(k + 7) % side] + 0.5}} for k in range(side)}
    if side <= mot_eval.MAX_CLEAR_COMPONENT:
        _, summary, _ = _evaluate({"clump": (results, frames)})
        assert summary["num_misses"]["clump"] == 0
        out, _ = mot_eval.evaluate_counters([mot_eval.get_mot_accum(results, frames)])
        assert out[0, 11] == side and out[0, 12] == side
    else:
        with pytest.raises(RuntimeError, match="residual assignment has a component over 64"):
            mot_eval.evaluate_mot_accums([mot_eval.get_mot_accum(results, frames)], ["clump"])


@pytest.mark.parametrize("n", [mot_eval.MAX_ID_COMPONENT[0], mot_eval.MAX_ID_COMPONENT[0] + 1])
def test_identity_component_limit_smaller_side(dev, n):
    """n GT ids and n tracks in one tp component (a ring): GT k meets track k, and in a later frame track k + 1 (mod
    n), on a grid of 1,024 boxes per frame"""
    boxes = _grid_boxes(1024).astype(np.float32)
    frames, results = [], {}
    for shift in (0, 1):
        for c in range(0, n, 1024):
            ks = range(c, min(n, c + 1024))
            frames.append({"gt": {k: boxes[k - c] for k in ks}})
            for k in ks:
                results.setdefault((k + shift) % n, {})[len(frames) - 1] = {"bbox": boxes[k - c]}
    acc = mot_eval.get_mot_accum(results, frames)
    if n > mot_eval.MAX_ID_COMPONENT[0]:
        with pytest.raises(RuntimeError, match="identity matching has a component over 8192 x 65536"):
            mot_eval.evaluate_mot_accums([acc], ["ring"])
        return
    summary, _ = mot_eval.evaluate_mot_accums([acc], ["ring"])
    t0 = time.perf_counter()
    out, _ = mot_eval.evaluate_counters([acc])
    print(f"ring {n} x {n}: evaluate_counters {1e3 * (time.perf_counter() - t0):.1f} ms")
    assert (out[0, 13], out[0, 14], out[0, 10]) == (n, n, n)               # one component; IDTP = n
    s = summary.loc["ring"]
    assert (s["num_switches"], s["num_misses"], s["num_false_positives"], s["mostly_tracked"]) == (n, 0, 0, n)


@pytest.mark.parametrize("extra", [0, 1])
def test_identity_component_limit_larger_side(dev, extra):
    """one GT id met by 64 fresh tracks in each of 1,024 frames: a 1 x 65,536 tp component (plus `extra` tracks)"""
    rng = np.random.default_rng(3)
    gt = np.asarray([100, 100, 200, 300], np.float32)
    n_frames = 1024 + extra
    frames = [{"gt": {1: gt}} for _ in range(n_frames)]
    results, t = {}, 0
    for f in range(n_frames):
        for _ in range(64 if f < 1024 else extra):
            results[t] = {f: {"bbox": (gt + rng.uniform(0, 1, 4)).astype(np.float32)}}
            t += 1
    acc = mot_eval.get_mot_accum(results, frames)
    if extra:
        with pytest.raises(RuntimeError, match="identity matching has a component over"):
            mot_eval.evaluate_mot_accums([acc], ["star"])
        return
    summary, _ = mot_eval.evaluate_mot_accums([acc], ["star"])
    t0 = time.perf_counter()
    out, _ = mot_eval.evaluate_counters([acc])
    print(f"star 1 x 65536: evaluate_counters {1e3 * (time.perf_counter() - t0):.1f} ms")
    assert (out[0, 13], out[0, 14], out[0, 10]) == (1, 65536, 1)
    s = summary.loc["star"]
    assert (s["num_switches"], s["num_misses"], s["num_false_positives"]) == (1023, 0, 63 * 1024)


def test_track_sequences_end_to_end(dev):
    """the scripted sequences tracked together by MultiSequenceTracker, scored against their scenes' objects"""
    import multi_tracker_fixtures as mtf
    import tracker_fixtures as tf
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.multi_tracker import MultiSequenceTracker, track_sequences
    specs = mtf.sequence_specs(6, noise=False)
    dets = [make().to(dev) for _, make, _, _ in specs]
    tr = MultiSequenceTracker(mtf.Mux(dets).to(dev), {"bbox": DeformablePostProcess()}, tf.BASE_CFG, max_batch=3)
    with torch.no_grad():
        results = track_sequences(tr, {s: mtf.blobs(det, s, frames, public, dev)
                                       for s, ((_, _, frames, public), det) in enumerate(zip(specs, dets))})
    named = {}
    for s, ((_, _, n_frames, _), det) in enumerate(zip(specs, dets)):
        sc = det.scene
        frames = []
        for t in range(n_frames):
            gt = {}
            for j in range(sc.n):
                if sc.alive(j, t):
                    cx, cy, w, h = sc.box(j, t)
                    gt[j] = np.asarray([(cx - w / 2) * tf.IMG_W, (cy - h / 2) * tf.IMG_H, (cx + w / 2) * tf.IMG_W,
                                        (cy + h / 2) * tf.IMG_H], np.float32)
            frames.append({"gt": gt})
        named[f"seq{s}"] = (results[s], frames)
    _, summary, text = _evaluate(named)
    print(text)
    assert summary["num_misses"]["OVERALL"] < summary["num_unique_objects"]["OVERALL"] * tf.N_FRAMES
    assert (summary["recall"].drop("OVERALL") > 0.3).all()
