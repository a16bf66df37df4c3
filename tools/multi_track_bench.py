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

`--model mots`: the MOTS workload.  The vanilla DETRSegmTracking (`vanilla_args(tracking=True, masks=True,
dataset="mot")`, random weights, class 0 pushed as above, the query embedding scaled by 100 so that the scores of
different queries differ by more than float noise; the first-frame threshold takes the widest gap between --tracks / 2
and 2 --tracks started tracks) tracks four sequences shaped like MOTS20, three at 1080x1920
and one at 480x640 (two input-size groups per step), with segmentation masks (bool, or COCO RLEs with `--mask-rle`) and,
with `--attention-maps`, the decoder attention maps.  Random weights make masks of many short runs, so the mask and RLE
work per frame is larger than a trained model's.  `--batches` defaults to 1,4 there.

`--check` runs every arm once over a few frames and asserts that each sequence got the same track ids and frame sets
from every arm (for MOTS it also prints the lowest mask IoU of any result against the serial arm's).  `--profile`
instead traces `--frames` steps of each arm in a separate `torch.profiler` run and reports, per step, the
device-to-host copies, the host's stream synchronises (read-backs and blocking copies), the frame ingest's waits for
its staging buffer (a second frame of the same size in one step waits for the first one's upload) and the project's
kernel launches (`msda_b200_launch_count`).  Prints one JSON line.  Not a bench.py arm.
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
    ap.add_argument("--model", choices=["deformable", "multi_frame", "mots"], default="deformable")
    ap.add_argument("--sequences", type=int, default=8, help="(mots: always the four MOTS20-shaped sequences)")
    ap.add_argument("--frames", type=int, default=12, help="timed frames per sequence and window")
    ap.add_argument("--warmup", type=int, default=3, help="untimed frames per sequence before each window")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--tracks", type=int, default=None, help="tracks each sequence starts (default 50; mots 20)")
    ap.add_argument("--batches", default=None, help="default 1,2,4,8; mots 1,4")
    ap.add_argument("--bucket", type=int, default=32)
    ap.add_argument("--mask-rle", action="store_true", help="mots: results' masks as COCO RLEs")
    ap.add_argument("--attention-maps", action="store_true", help="mots: generate the decoder attention maps")
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    mots = args.model == "mots"
    args.tracks = args.tracks or (20 if mots else 50)
    args.batches = args.batches or ("1,4" if mots else "1,2,4,8")
    from trackformer_b200.deformable_detr import DeformablePostProcess, PostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.frame_ingest import FrameIngest
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args, vanilla_args
    from trackformer_b200.multi_tracker import MultiSequenceTracker
    from trackformer_b200.segmentation import PostProcessSegm

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    if mots:
        model, _, _ = build_model(vanilla_args(tracking=True, masks=True, dataset="mot", device="cuda:0"))
    else:
        model, _, _ = build_model(default_args(True, args.model == "multi_frame", device="cuda:0"))
    with torch.no_grad():
        for name, p in model.named_parameters():               # make class 0 the winning label (random weights)
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 8.0
        if mots:            # random vanilla decoder rows differ by ~1e-4 (scores within float noise): spread them
            model.query_embed.weight.mul_(100.0)
    model.to(dev).eval()
    model.tracking()
    rng = np.random.default_rng(1)
    shapes = [(1080, 1920)] * 3 + [(480, 640)] if mots else [(1080, 1920)] * args.sequences
    args.sequences = len(shapes)
    videos = [[rng.integers(0, 256, shape + (3,), dtype=np.uint8) for _ in range(4)] for shape in shapes]
    base = dict(public_detections=False, detection_obj_score_thresh=2.0, track_obj_score_thresh=-1.0,
                detection_nms_thresh=0.0, track_nms_thresh=0.0, steps_termination=1, prev_frame_dist=1,
                inactive_patience=-1, reid_sim_threshold=0.0, reid_sim_only=False, reid_score_thresh=2.0,
                reid_greedy_matching=False)
    post = PostProcess() if mots else DeformablePostProcess()
    posts = {"bbox": post, "segm": PostProcessSegm()} if mots else {"bbox": post}
    extra = dict(generate_attention_maps=args.attention_maps, mask_rle=args.mask_rle) if mots else {}
    ingest = FrameIngest(dev)
    first_thresh, first_gap = [], []
    with torch.no_grad():                                       # per sequence: the threshold that starts --tracks
        for video in videos:
            blob = ingest(video[0])
            detect = model.detect if mots else model
            rows = post.packed(detect(blob["img"], None, None)[0], blob["orig_size"].to(dev))[0].cpu().numpy()
            s = np.sort(rows[rows[:, 1] == 0, 0])[::-1]
            # the widest gap near --tracks; MOTS searches wider (tracks / 2 .. 2 tracks): random vanilla scores are
            # packed so densely that batch-size noise could move a decision across a narrow gap
            lo, hi = (args.tracks // 2, min(2 * args.tracks, len(s) - 1)) if mots else (args.tracks - 3, args.tracks + 3)
            gaps = s[lo:hi] - s[lo + 1:hi + 1]
            k = lo + int(np.argmax(gaps))
            first_thresh.append(float((s[k] + s[k + 1]) / 2))
            first_gap.append(float(s[k] - s[k + 1]))

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
                trs = [DeviceTracker(a["det"], posts, cfg(i, 0), frame_ingest=ingest, **extra)
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
                tr = MultiSequenceTracker(a["det"], posts, base, max_batch=b, frame_ingest=ingest, **extra)
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
            "input": ("3 x 1080x1920 + 1 x 480x640 uint8" if mots else "1080x1920 uint8 -> 750x1333"),
            "tracks": args.tracks}
    if mots:
        line.update(mask_rle=args.mask_rle, attention_maps=args.attention_maps,
                    note="random weights: masks of many short runs")
    if args.check:
        from trackformer_b200.mots import decode
        ref, ref_res, lowest = None, None, 1.0
        for arm in arms:
            res = run(arm, 0, 6)
            summary = {i: {tid: sorted(r[tid]) for tid in r} for i, r in res.items()}
            assert all(len(s) > 0 for s in summary.values()), arm
            if ref is None:
                ref, ref_res = summary, res
            differ = [i for i in summary if summary[i] != ref[i]]
            if differ:
                line.setdefault("differ", {})[arm] = {
                    i: {"ids": [len(summary[i]), len(ref[i])],
                        "first_frame_ids": [sum(0 in f for f in summary[i].values()),
                                            sum(0 in f for f in ref[i].values())]} for i in differ}
                continue
            if mots and res is not ref_res:
                for i, r in res.items():
                    for tid, frames in r.items():
                        for f, e in frames.items():
                            m, w = e["mask"], ref_res[i][tid][f]["mask"]
                            m, w = (decode(x) if isinstance(x, dict) else np.asarray(x) for x in (m, w))
                            union = int((m | w).sum())
                            lowest = min(lowest, 1.0 if union == 0 else int((m & w).sum()) / union)
        line["first_frame_threshold_gap_min"] = min(first_gap)
        if mots:
            line["lowest_mask_iou_vs_serial"] = round(lowest, 6)
        line["check"] = "same track ids and frame sets in every arm" if "differ" not in line else "FAILED"
        print(json.dumps(line))
        assert "differ" not in line, "an arm tracked differently from serial"
        return
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        import ctypes
        from trackformer_b200 import ext
        counter = ctypes.CDLL(ext.library_path()).msda_b200_launch_count
        counter.restype = ctypes.c_int64
        for arm in arms:
            run(arm, args.warmup, 1)                            # captures and buffers outside the trace
            steps_before = len(arms[arm]["times"])
            launches = int(counter())
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                run(arm, 0, args.frames)
            launches = int(counter()) - launches
            steps = len(arms[arm]["times"]) - steps_before
            events = prof.events()
            dtoh = sum(1 for e in events if "DtoH" in e.name or "Device -> Pageable" in e.name
                       or "Device -> Pinned" in e.name)
            def calls(name):
                return sum(1 for e in events if e.name == name)
            # the step timer's own two device synchronises are not the tracker's
            device = calls("cudaDeviceSynchronize") - 2 * steps
            line[arm] = {"steps": steps, "dtoh_copies_per_step": round(dtoh / steps, 2),
                         "stream_syncs_per_step": round((calls("cudaStreamSynchronize") + device) / steps, 2),
                         "ingest_staging_waits_per_step": round(calls("cudaEventSynchronize") / steps, 2),
                         "project_launches_per_step": round(launches / steps, 2)}
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
