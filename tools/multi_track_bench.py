#!/usr/bin/env python
"""Throughput of tracking several sequences at once: N serial DeviceTrackers vs MultiSequenceTracker at B = 1, 2, 4, 8.

Workload: `--sequences` synthetic uint8 1080x1920 videos (each its own four random frames, host numpy arrays like a
decoder's output), ingested on the device to 750x1333, tracked by the deformable tracking model (`--model
deformable`, 300 queries) or the multi-frame model (`--model multi_frame`, 500 queries, hidden 288).  Random weights
with class 0 made the winner; each sequence's first frame starts `--tracks` tracks (a threshold between two of its
scores), after which every track is kept and none starts, so all arms carry the same load.

Arms: `serial` -- one DeviceTracker per sequence over one shared GraphedDetector, the sequences stepped one after the
other each frame (the per-sequence loop of src/track.py); `B=b` -- MultiSequenceTracker(max_batch=b), the sequences
in rounds of b stepped together.  The arms alternate over `--windows` windows; per arm the line gives aggregate
frames/s (all frames over all timed steps' time), the per-step latency (median, p10-p90; a step is one tracker call:
one sequence's frame for `serial`, b sequences' frames for `B=b`), the graph captures and the peak memory allocated while the
arm ran, above what was allocated when it started (the first window includes its graph captures).
The card's name and power limit are read in the same run.

`--check` runs every arm once over a few frames and asserts that each sequence got the same track ids and frame sets
from every arm.  Prints one JSON line.  Not a bench.py arm.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                        text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["deformable", "multi_frame"], default="deformable")
    ap.add_argument("--sequences", type=int, default=8)
    ap.add_argument("--frames", type=int, default=12, help="timed frames per sequence and window")
    ap.add_argument("--warmup", type=int, default=3, help="untimed frames per sequence before each window")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--tracks", type=int, default=50)
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--bucket", type=int, default=32)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.frame_ingest import FrameIngest
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.multi_tracker import MultiSequenceTracker

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model, _, _ = build_model(default_args(True, args.model == "multi_frame", device="cuda:0"))
    with torch.no_grad():
        for name, p in model.named_parameters():               # make class 0 the winning label (random weights)
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 8.0
    model.to(dev).eval()
    model.tracking()
    rng = np.random.default_rng(1)
    videos = [[rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8) for _ in range(4)] for _ in range(args.sequences)]
    base = dict(public_detections=False, detection_obj_score_thresh=2.0, track_obj_score_thresh=-1.0,
                detection_nms_thresh=0.0, track_nms_thresh=0.0, steps_termination=1, prev_frame_dist=1,
                inactive_patience=-1, reid_sim_threshold=0.0, reid_sim_only=False, reid_score_thresh=2.0,
                reid_greedy_matching=False)
    post = DeformablePostProcess()
    ingest = FrameIngest(dev)
    first_thresh = []
    with torch.no_grad():                                       # per sequence: the threshold that starts --tracks
        for video in videos:
            blob = ingest(video[0])
            rows = post.packed(model(blob["img"], None, None)[0], blob["orig_size"].to(dev))[0].cpu().numpy()
            s = np.sort(rows[rows[:, 1] == 0, 0])[::-1]
            gaps = s[args.tracks - 3:args.tracks + 3] - s[args.tracks - 2:args.tracks + 4]
            k = args.tracks - 3 + int(np.argmax(gaps))
            first_thresh.append(float((s[k] + s[k + 1]) / 2))

    def blob(i, t):
        return {"frame": videos[i][t % 4]}

    def cfg(i, t):
        return dict(base, detection_obj_score_thresh=first_thresh[i] if t == 0 else 2.0)

    def set_thresh(tr, i, t):
        tr.detection_obj_score_thresh = first_thresh[i] if t == 0 else 2.0

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    arms = {"serial": {"det": GraphedDetector(model, bucket=args.bucket)}}
    for b in (int(x) for x in args.batches.split(",")):
        arms[f"B={b}"] = {"det": GraphedDetector(model, bucket=args.bucket), "b": b}
    for a in arms.values():
        a.update(times=[], frames=0, seconds=0.0, peak=0)

    def run(name, n_warm, n_timed):
        """every sequence from its first frame: n_warm untimed frames, then n_timed timed ones; returns results"""
        a = arms[name]
        torch.cuda.reset_peak_memory_stats()
        start_alloc = torch.cuda.memory_allocated()
        results = {}
        with torch.no_grad():
            if name == "serial":
                trs = [DeviceTracker(a["det"], {"bbox": post}, cfg(i, 0), False, frame_ingest=ingest)
                       for i in range(args.sequences)]
                for t in range(n_warm + n_timed):
                    for i, tr in enumerate(trs):
                        set_thresh(tr, i, t)
                        ms = timed(lambda: tr.step(blob(i, t)))
                        if t >= n_warm:
                            a["times"].append(ms)
                            a["frames"] += 1
                            a["seconds"] += ms / 1e3
                results = {i: tr.results for i, tr in enumerate(trs)}
            else:
                b = a["b"]
                tr = MultiSequenceTracker(a["det"], {"bbox": post}, base, max_batch=b, frame_ingest=ingest)
                for r0 in range(0, args.sequences, b):
                    group = range(r0, min(r0 + b, args.sequences))
                    for i in group:
                        tr.start(i, cfg(i, 0))
                    for t in range(n_warm + n_timed):
                        for i in group:
                            set_thresh(tr.sequence(i), i, t)
                        ms = timed(lambda: tr.step({i: blob(i, t) for i in group}))
                        if t >= n_warm:
                            a["times"].append(ms)
                            a["frames"] += len(group)
                            a["seconds"] += ms / 1e3
                    for i in group:
                        results[i] = tr.finish(i)
        a["peak"] = max(a["peak"], torch.cuda.max_memory_allocated() - start_alloc)
        return results

    name, power = card()
    line = {"card": name, "power_limit": power, "model": args.model, "sequences": args.sequences,
            "input": "1080x1920 uint8 -> 750x1333", "tracks": args.tracks}
    if args.check:
        ref = None
        for arm in arms:
            res = run(arm, 0, 6)
            summary = {i: {tid: sorted(r[tid]) for tid in r} for i, r in res.items()}
            assert all(len(s) > 0 for s in summary.values()), arm
            if ref is None:
                ref = summary
            assert summary == ref, f"arm {arm} tracked differently from serial"
        line["check"] = "same track ids and frame sets in every arm"
        print(json.dumps(line))
        return
    order = list(arms)
    for w in range(args.windows):
        for arm in (order if w % 2 == 0 else order[::-1]):
            run(arm, args.warmup, args.frames)
    for arm, a in arms.items():
        t = np.asarray(a["times"])
        line[arm] = {"frames_per_s": round(a["frames"] / a["seconds"], 1), "step_ms_median": round(float(np.median(t)), 2),
                     "step_ms_p10_p90": [round(float(np.percentile(t, 10)), 2), round(float(np.percentile(t, 90)), 2)],
                     "captures": a["det"].captures, "peak_alloc_above_start_GiB": round(a["peak"] / 2 ** 30, 2)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
