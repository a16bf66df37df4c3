#!/usr/bin/env python
"""Attention-map tracking fixtures recorded FROM THE REFERENCE (build container only).

Runs the unmodified reference `Tracker(..., generate_attention_maps=True)` (src/trackformer/models/tracker.py:37-60,
335-481, 539-541) over the reference DETRSegmTracking (cfgs/train.yaml, train_tracking.yaml, ``masks: true``) on CPU,
with the canonical weights and class-0 bias push of tests/tracker_fixtures.py and the score spreading of
tests/attention_map_fixtures.py (``condition_``), on a 256 x 320 'video' (8 x 10 maps).
The random box head puts every box on nearly the same spot, so NMS is off (it would keep one track).  The detection
threshold is placed inside a gap of the first frame's object-query scores, the track and ReID thresholds inside the
lower band of the track-query scores, and ReID by embedding distance is off (``reid_sim_threshold`` 0), so a track
that is present in two consecutive frames was kept through its own track query and a track that comes back after a
missing frame was re-identified through its track query.  Among a small grid, the run kept is the one that has all of
these events -- tracks kept through their track queries, tracks inactive for a frame or more that come back, and
track-query counts in more than one bucket of 3 (GraphedDetector's padding) -- with the widest score margin (track
rows against the track / ReID thresholds, object rows against the detection threshold).  Stores:

  * tracker_attention_maps.npz       box post-processing only
  * tracker_attention_maps_segm.npz  box + mask post-processing (PostProcessSegm)

each with the summary rows, ``map_keys`` (id, frame), ``maps`` [N, 8, 10] float32, ``n_queries`` (track queries per
frame), the tracker cfg, ``class_bias`` and ``margin``.  The masks enter no tracking decision and the summary holds no
mask, so the two files are expected to be equal: the second pins that the mask post-processing leaves the decisions and
maps alone.

The reference's box-only DETRTracking cannot be recorded: its hook reads the layer-4 size from backbone output '3',
which only a backbone returning intermediate layers (masks) produces.  The vanilla models need the ``prev_features``
shim of make_golden_detr.py.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
sys.path.insert(0, HERE)


def main():
    import torch
    import yaml
    from make_golden_model import import_reference
    from make_golden_detr import drop_prev_features, REF
    build_model, to_ns = import_reference()
    import trackformer.models.detr as detr
    import trackformer.models.detr_segmentation as seg
    from trackformer.models.tracker import Tracker
    drop_prev_features(detr.DETR)
    drop_prev_features(seg.DETRSegmBase)
    import attention_map_fixtures as amf

    def build(tracking, multi_frame, **overrides):
        assert tracking and not multi_frame
        cfg = yaml.safe_load(open(os.path.join(REF, "cfgs", "train.yaml")))
        cfg.update(yaml.safe_load(open(os.path.join(REF, "cfgs", "train_tracking.yaml"))))
        cfg["dataset"] = "mot"
        cfg["device"] = "cpu"
        cfg.update(overrides)
        torch.manual_seed(0)
        model, criterion, _ = build_model(to_ns(cfg))
        return model, criterion

    class_bias = amf.condition_(build(True, False, masks=True)[0])

    def run(cfg, segm, log=None):
        post = detr.PostProcess()
        if log is not None:
            inner = post

            class Logged:
                def __call__(self, outputs, sizes):
                    res = inner(outputs, sizes)
                    log.append((res[0]["scores"].numpy().copy(), res[0]["labels"].numpy().copy()))
                    return res
            post = Logged()
        posts = {"bbox": post}
        if segm:
            posts["segm"] = seg.PostProcessSegm()
        return amf.run_sequence(build, Tracker, posts, cfg, class_bias)

    probe_log = []
    run(dict(detection_obj_score_thresh=2.0), False, probe_log)
    s0 = np.sort(probe_log[0][0][probe_log[0][1] == 0])[::-1]
    best = None
    for k in range(3, 6):
        thr = float((s0[k] + s0[k + 1]) / 2)
        for t_track, d_reid in ((0.6, -0.04), (0.64, -0.04), (0.64, -0.08), (0.68, -0.04), (0.68, -0.08), (0.72, -0.06)):
            cfg = dict(detection_obj_score_thresh=thr, track_obj_score_thresh=t_track, reid_score_thresh=t_track + d_reid,
                       inactive_patience=3, reid_sim_threshold=0.0, detection_nms_thresh=0.0, track_nms_thresh=0.0,
                       steps_termination=1)
            log = []
            out = run(cfg, False, log)
            events = amf.events(out)
            gaps = []
            for (sc, _), nq in zip(log, out["n_queries"]):
                gaps.append(np.abs(sc[nq:] - thr).min())
                if nq:
                    gaps += [np.abs(sc[:nq] - cfg["track_obj_score_thresh"]).min(),
                             np.abs(sc[:nq] - cfg["reid_score_thresh"]).min()]
            margin = float(min(gaps))
            print(f"k={k} track={t_track} reid={t_track + d_reid:.2f}: margin={margin:.2e} rows={len(out['rows'])} "
                  f"events={events} reids={int(out['num_reids'])} track_num={int(out['track_num'])}", flush=True)
            if all(events.values()) and (best is None or margin > best[0]):
                best = (margin, cfg, out, thr)
    margin, cfg, out, thr = best
    for name, segm in (("tracker_attention_maps", False), ("tracker_attention_maps_segm", True)):
        res = out if not segm else run(cfg, True)
        res["cfg_keys"] = np.asarray(sorted(cfg))
        res["cfg_values"] = np.asarray([cfg[k] for k in sorted(cfg)], np.float64)
        res["margin"] = np.float64(margin)
        res["class_bias"] = class_bias
        np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **res)
        print(f"{name}: thr={thr:.6f} margin={margin:.2e} rows={len(res['rows'])} maps={res['maps'].shape} "
              f"ids={sorted(set(res['rows'][:, 0].astype(int)))} reids={int(res['num_reids'])} "
              f"active={res['active_ids'].tolist()} inactive={res['inactive_ids'].tolist()} "
              f"map sums {res['maps'].sum((1, 2)).min():.6f}..{res['maps'].sum((1, 2)).max():.6f}", flush=True)


if __name__ == "__main__":
    main()
