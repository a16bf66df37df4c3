"""Attention-map tracking runs shared by the reference recorder (tests/golden/make_golden_attention_maps.py, build
container only) and the tests (test infrastructure).

``run_sequence`` drives a tracker class with ``generate_attention_maps=True`` over a vanilla tracking model --
DETRSegmTracking (``masks=True``) or DETRTracking -- set up like tracker_fixtures.run_model_sequence (canonical
weights, class-0 bias push), on the slowly changing random 'video' of tracker_fixtures.model_frames, and returns the
tracker summary plus every (id, frame) attention map of the results.

With canonical weights the vanilla decoder's output rows differ by ~1e-4 between queries, so every score sits within
1e-4 of the others and no threshold separates them by more than float noise.  ``condition_`` spreads them: the query
embedding is scaled by QUERY_SCALE (the rows then differ ~100x more) and ``class_embed`` by CLASS_SCALE around the mean
row of the first frame, whose bias (``class_bias``, recorded with the fixture) keeps that mean row's logits where the
class-0 push put them.  Object-query scores then spread over ~0.85 .. 0.9 and the labels mix; track-query rows (zero
query position, the previous embedding as content) score lower, ~0.6 .. 0.85, which is where the track and ReID
thresholds go.
"""
import numpy as np
import torch

import model_fixtures as mf
import tracker_fixtures as tf

SIZE = (256, 320)                          # stride-32 maps of 8 x 10
N_FRAMES = 8


QUERY_SCALE = 100.0
CLASS_SCALE = 10.0


def condition_(model, class_bias=None):
    """Canonical weights, the class-0 push and the score spreading described above.  ``class_bias`` None computes it
    from the model's own first-frame forward (the recorder); returns it."""
    mf.canonical_weights_(model, 0)
    with torch.no_grad():
        model.query_embed.weight.mul_(QUERY_SCALE)
        w, b = model.class_embed.weight, model.class_embed.bias
        if class_bias is None:
            model.eval()
            hs = model(next(blobs())["img"])[4][-1][0]            # last decoder layer, normed: the class head's input
            push = torch.zeros_like(b)
            push[0] = 6.0                  # random weights favour an arbitrary class: make it class 0 ("person")
            class_bias = (b + push - (CLASS_SCALE - 1.0) * (w @ hs.mean(0))).numpy()
        w.mul_(CLASS_SCALE)
        b.copy_(torch.as_tensor(np.asarray(class_bias), dtype=b.dtype))
    return np.asarray(class_bias, np.float32)


def build_tracker(build, tracker_cls, posts, cfg_overrides, class_bias, masks=True, device="cpu", wrap=None):
    model, _ = build(True, False, masks=masks)
    condition_(model, class_bias)
    model.to(device)
    model.tracking()
    cfg = dict(tf.BASE_CFG)
    cfg.update(cfg_overrides)
    tracker = tracker_cls(model if wrap is None else wrap(model), posts, cfg, True)
    tracker.reset()
    return tracker, model


def blobs(size=SIZE, n_frames=N_FRAMES):
    for frame in tf.model_frames(size, n_frames):
        yield {"img": frame[None], "orig_size": torch.tensor([list(size)]), "dets": torch.zeros(1, 0, 4),
               "size": torch.tensor([list(size)])}


def summarise(tracker):
    """tracker_fixtures.summarise plus ``map_keys`` [N, 2] (id, frame) and ``maps`` [N, h, w] in that order."""
    out = tf.summarise(tracker)
    keys, maps = [], []
    for tid in sorted(tracker.results):
        for frame in sorted(tracker.results[tid]):
            m = tracker.results[tid][frame].get("attention_map")
            if m is not None:
                keys.append([tid, frame])
                maps.append(np.asarray(m, np.float32))
    out["map_keys"] = np.asarray(keys, np.int64).reshape(-1, 2)
    out["maps"] = np.stack(maps) if maps else np.zeros((0, 1, 1), np.float32)
    return out


def run_sequence(build, tracker_cls, posts, cfg_overrides, class_bias, masks=True, device="cpu", wrap=None, size=SIZE,
                 n_frames=N_FRAMES):
    tracker, _ = build_tracker(build, tracker_cls, posts, cfg_overrides, class_bias, masks, device, wrap)
    n_queries = []
    with torch.no_grad():
        for blob in blobs(size, n_frames):
            n_queries.append(len(tracker.tracks) + len(tracker.inactive_tracks))      # track queries of this frame
            tracker.step(blob)
    out = summarise(tracker)
    out["n_queries"] = np.asarray(n_queries, np.int64)
    return out


def events(res):
    """What a run exercises, from its summary: ``kept`` -- an id present in two consecutive frames (with ReID by
    embedding distance off, only its own track query can carry it over); ``returned`` -- an id that is missing for a
    frame or more and then comes back (re-identified through its track query); ``buckets`` -- track-query counts in
    more than one nonzero bucket of 3."""
    frames = {}
    for tid, f in res["rows"][:, :2].astype(int):
        frames.setdefault(tid, []).append(f)
    steps = [b - a for fs in frames.values() for a, b in zip(sorted(fs), sorted(fs)[1:])]
    return {"kept": any(d == 1 for d in steps), "returned": any(d > 1 for d in steps),
            "buckets": len({-(-int(n) // 3) for n in res["n_queries"] if n}) > 1}


def golden_cfg(gold):
    return {str(k): (int(v) if k == "steps_termination" else float(v)) for k, v in zip(gold["cfg_keys"], gold["cfg_values"])}
