#!/usr/bin/env python
"""Online-tracking latency on one GPU: Tracker.step per frame, eager detector vs CUDA-graph replay.

Workload (SURVEY section 8, config C3): tracking model (deformable DETR R50, 20-class head), one 3x800x1333 frame per
step, `--tracks` live track queries (default 100) + 300 object queries, random-init weights, synthetic frames.  Each
timed step is the whole `Tracker.step(blob)`: host frame -> device, forward, fused post-processing, one read-back, host
bookkeeping.  Random weights give flat scores, so the live-track count is pinned by thresholds: the first frame starts
exactly `--tracks` tracks, afterwards every track is kept and no new ones start.

`--masks` tracks with the segmentation model (DeformableDETRSegmTracking, "segm" post-processing): Tracker and
DeviceTracker over the CUDA-graph detector, each running the mask head on the rows the frame's decisions keep and
resolving the masks into one label map, against the reference-shaped work for the same frame -- the full forward with
`pred_masks` for every query row plus PostProcessSegm(return_probs=True), which upsamples every row to the image and
copies it to the host.  Each tracker runs twice, frame by frame in turn: with the results' bool masks (the label map
read back) and with `mask_rle=True` (COCO RLE strings made on the device); per arm the line gives the latency, the
device-to-host bytes of the masks per frame as counted from what arrived, and the host bytes the results' masks hold
at the end (bool arrays' nbytes against the strings' lengths).

Prints one JSON line; tools/README.md lists it among the measurement aids.  Not a bench.py arm.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=100)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--height", type=int, default=800)
    ap.add_argument("--width", type=int, default=1333)
    ap.add_argument("--multi-frame", action="store_true")
    ap.add_argument("--bucket", type=int, default=32)
    ap.add_argument("--no-tf32", action="store_true")
    ap.add_argument("--skip-eager", action="store_true", help="only the CUDA-graph detector")
    ap.add_argument("--masks", action="store_true", help="segmentation model, tracking with masks")
    args = ap.parse_args()
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.tracker import Tracker

    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = not args.no_tf32
    torch.manual_seed(0)
    model, _, _ = build_model(default_args(True, args.multi_frame, device="cuda:0", **({"masks": True} if args.masks else {})))
    with torch.no_grad():
        for name, p in model.named_parameters():               # make class 0 the winning label (random weights)
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 8.0
    model.to(dev).eval()
    model.tracking()
    g = torch.Generator().manual_seed(1)
    frames = [torch.randn(1, 3, args.height, args.width, generator=g).pin_memory() for _ in range(4)]
    cfg = dict(public_detections=False, detection_obj_score_thresh=2.0, track_obj_score_thresh=-1.0,
               detection_nms_thresh=0.0, track_nms_thresh=0.0, steps_termination=1, prev_frame_dist=1,
               inactive_patience=-1, reid_sim_threshold=0.0, reid_sim_only=False, reid_score_thresh=2.0,
               reid_greedy_matching=False)
    size = torch.tensor([[args.height, args.width]])

    def blob(i):
        b = {"img": frames[i % 4], "orig_size": size, "dets": torch.zeros(1, 0, 4)}
        if args.masks:
            b["size"] = size
        return b

    def start(detector, tracker_cls=Tracker, **kwargs):
        """a tracker whose first frame starts exactly --tracks tracks"""
        post = DeformablePostProcess()
        posts = {"bbox": post}
        if args.masks:
            from trackformer_b200.segmentation import PostProcessSegm
            posts["segm"] = PostProcessSegm()
        tr = tracker_cls(detector, posts, cfg, False, **kwargs)
        tr.reset()
        with torch.no_grad():
            out = detector(frames[0].to(dev), None, None)[0]
        rows = post.packed(out, size.to(dev))[0].cpu().numpy()
        s = np.sort(rows[rows[:, 1] == 0, 0])[::-1]
        assert len(s) > args.tracks, "not enough class-0 queries to start the requested number of tracks"
        tr.detection_obj_score_thresh = float((s[args.tracks - 1] + s[args.tracks]) / 2)
        tr.step(blob(0))
        tr.detection_obj_score_thresh = 2.0
        assert len(tr.tracks) == args.tracks, len(tr.tracks)
        return tr

    def timed_step(tr, i):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tr.step(blob(i + 1))
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    def run(detector, tracker_cls=Tracker):
        tr = start(detector, tracker_cls)
        times = []
        for i in range(args.warmup + args.frames):
            t = timed_step(tr, i)
            if i >= args.warmup:
                times.append(t)
        assert len(tr.tracks) == args.tracks
        return times

    if args.masks:
        print(json.dumps(masks_line(args, model, frames, size, dev, start, timed_step)))
        return
    det = GraphedDetector(model, bucket=args.bucket)
    graphed = run(det)
    eager = graphed if args.skip_eager else run(model)
    device = run(GraphedDetector(model, bucket=args.bucket), DeviceTracker)      # decisions in csrc/track_step.cu
    line = {
        "what": "Tracker.step latency, host frame in -> results out", "frames": args.frames, "warmup": args.warmup,
        "config": {"workload": f"tracking{' multi-frame' if args.multi_frame else ''} 1x3x{args.height}x{args.width}, "
                               f"{args.tracks} track + {model.num_queries} object queries", "bucket": args.bucket,
                   "tf32": not args.no_tf32},
        "eager_ms": {"median": float(np.median(eager)), "p10": float(np.percentile(eager, 10)), "p90": float(np.percentile(eager, 90))},
        "graph_ms": {"median": float(np.median(graphed)), "p10": float(np.percentile(graphed, 10)), "p90": float(np.percentile(graphed, 90))},
        "graph_device_tracker_ms": {"median": float(np.median(device)), "p10": float(np.percentile(device, 10)),
                                    "p90": float(np.percentile(device, 90))},
        "eager_fps": 1e3 / float(np.median(eager)), "graph_fps": 1e3 / float(np.median(graphed)),
        "graph_device_tracker_fps": 1e3 / float(np.median(device)),
        "graph_captures": det.captures, "graph_replays": det.replays,
        "h2d_bytes_per_frame": int(frames[0].numel() * 4), "d2h_bytes_per_frame": int((args.tracks + model.num_queries) * 6 * 4),
        "d2h_bytes_per_frame_device_tracker": int((8 + 8 * (args.tracks + model.num_queries)) * 4),
    }
    print(json.dumps(line))


def masks_line(args, model, frames, size, dev, start, timed_step):
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.segmentation import PostProcessSegm
    from trackformer_b200.tracker import Tracker

    # the reference-shaped work of one frame: full forward (pred_masks for all rows) + PostProcessSegm to the host
    post = PostProcessSegm()
    with torch.no_grad():
        out, _, feats, _, _ = model(frames[0].to(dev), None, None)
        tgt = [{"track_query_boxes": out["pred_boxes"][0, :args.tracks].clone(),
                "track_query_hs_embeds": out["hs_embed"][0, :args.tracks].clone(),
                "image_id": torch.tensor([1], device=dev)}]
        full = []
        for i in range(args.warmup + args.frames):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            o, _, feats, _, _ = model(frames[(i + 1) % 4].to(dev), tgt, feats)
            post([{}], o, size.to(dev), size.to(dev), return_probs=True)
            torch.cuda.synchronize()
            if i >= args.warmup:
                full.append((time.perf_counter() - t0) * 1e3)
        n_rows = args.tracks + model.num_queries
        del out, o
    torch.cuda.empty_cache()

    # four arms -- {Tracker, DeviceTracker} x {bool masks, RLE masks} -- each over its own CUDA-graph detector, stepped
    # in turn frame by frame so that they share the machine's state
    arms = {}
    for name, cls, rle in (("graph_masks", Tracker, False), ("graph_masks_rle", Tracker, True),
                           ("graph_device_tracker_masks", DeviceTracker, False),
                           ("graph_device_tracker_masks_rle", DeviceTracker, True)):
        arms[name] = {"tracker": start(GraphedDetector(model, bucket=args.bucket), cls, mask_rle=rle), "rle": rle,
                      "times": [], "d2h": []}
    label_bytes = args.height * args.width * 4
    for i in range(args.warmup + args.frames):
        for arm in arms.values():
            tr = arm["tracker"]
            t = timed_step(tr, i)
            if i < args.warmup:
                continue
            arm["times"].append(t)
            # device-to-host bytes of the frame's masks, counted from what arrived: the label map, or the RLE header
            # (status, total, offset and length per result) plus the strings
            frame = [r[tr.frame_index - 1] for r in tr.results.values() if tr.frame_index - 1 in r]
            if arm["rle"]:
                arm["d2h"].append(8 * (2 + 2 * len(frame)) + sum(len(e["mask"]["counts"]) for e in frame))
            else:
                arm["d2h"].append(label_bytes)
    rows_d2h = {False: n_rows * 6 * 4, True: (8 + 8 * n_rows) * 4}        # the frame's result rows, per tracker kind

    def stats(t):
        return {"median": float(np.median(t)), "p10": float(np.percentile(t, 10)), "p90": float(np.percentile(t, 90))}
    line = {
        "what": "Tracker.step latency with segmentation masks, host frame in -> results (with masks) out",
        "frames": args.frames, "warmup": args.warmup,
        "config": {"workload": f"segmentation tracking 1x3x{args.height}x{args.width}, {args.tracks} track + "
                               f"{model.num_queries} object queries", "bucket": args.bucket, "tf32": not args.no_tf32},
        "reference_shaped_forward_plus_postprocess_segm_ms": stats(full),
        "head_rows_reference_shaped": n_rows,
        "d2h_bytes_per_frame_reference_shaped": int(n_rows * args.height * args.width * 4),
    }
    for name, arm in arms.items():
        tr = arm["tracker"]
        assert len(tr.tracks) == args.tracks
        held = sum(len(e["mask"]["counts"]) if arm["rle"] else e["mask"].nbytes
                   for r in tr.results.values() for e in r.values())
        line[name] = {"ms": stats(arm["times"]), "head_rows_last_frame": int((tr._result_rows >= 0).sum()),
                      "mask_d2h_bytes_per_frame": stats(arm["d2h"]),
                      "d2h_bytes_per_frame": float(np.median(arm["d2h"])) + rows_d2h[isinstance(tr, DeviceTracker)],
                      "results_mask_host_bytes": int(held), "results_frames": tr.frame_index}
    return line


if __name__ == "__main__":
    main()
