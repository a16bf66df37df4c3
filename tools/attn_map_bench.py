#!/usr/bin/env python
"""Cost of the tracker's attention maps (generate_attention_maps) on one GPU.

`kernel`: the head-averaged weights kernel (csrc/dense_attn.cu dense_attn_weights_kernel) alone at 300 / 400 query
rows x 1050 / 1008 / 4200 keys (8 heads of 32 channels, batch 1), next to the stock nn.MultiheadAttention(256, 8) with
need_weights=True and to the dense-attention replacement with and without need_weights on the same inputs.  Every
arm is captured in a CUDA graph of `--launches` calls and timed with CUDA events over `--repeats` replays, the arms
alternated; medians in microseconds per call.

`track`: Tracker.step and DeviceTracker.step over GraphedDetector for DETRSegmTracking (box post-processing, random
weights with the class-0 push) at 800 x 1333, with the maps on and off, the four arms stepped in turn frame by frame;
every object query starts a track in the first frame and no track starts afterwards (flat random-weight scores), so
each frame runs 100 track + 100 object queries; median ms per step, and the bytes of maps read back per frame (rows
that took a new map x h x w x 4).  Each step is also split, with a device synchronise around each part: the detector
call (graph replay + output slicing), the map gather and read-back (`_attention_maps`), and the rest of the step.

Prints one JSON line with the card name and power limit; stops without a CUDA device.  Not a bench.py arm.
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
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return name, limit
    except Exception:                                        # noqa: BLE001 -- the numbers still stand without it
        return torch.cuda.get_device_name(0), "unknown"


def graph_of(fn, launches):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            fn()
    return g


def kernel_part(args, dev):
    from trackformer_b200 import dense_attention, ext
    m = ext.load()
    res = []
    torch.manual_seed(0)
    mha = torch.nn.MultiheadAttention(256, 8).to(dev).eval()
    for lq in (300, 400):
        for lk in (1050, 1008, 4200):
            tgt = torch.randn(lq, 1, 256, device=dev)
            mem = torch.randn(lk, 1, 256, device=dev)
            qp = torch.randn(lq, 1, 512, device=dev)
            kv = torch.randn(lk, 1, 768, device=dev)
            q, k, v = qp[..., :256].unflatten(-1, (8, 32)), kv[..., 256:512].unflatten(-1, (8, 32)), \
                kv[..., 512:].unflatten(-1, (8, 32))
            scale = 32 ** -0.5
            _, lse = m.dense_attention_forward(q, k, v, None, None, scale, 1.0)
            with torch.no_grad():
                arms = {
                    "weights_kernel": lambda: m.dense_attention_weights(q, k, None, lse, scale),
                    "attention_need_weights": lambda: dense_attention.attention(mha, tgt, mem, mem, None, True),
                    "attention": lambda: dense_attention.attention(mha, tgt, mem, mem, None),
                    "stock_need_weights": lambda: mha(tgt, mem, mem, need_weights=True),
                }
                graphs = {name: graph_of(fn, args.launches) for name, fn in arms.items()}
            times = {name: [] for name in arms}
            for _ in range(args.repeats):
                for name, g in graphs.items():
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    g.replay()
                    b.record()
                    b.synchronize()
                    times[name].append(a.elapsed_time(b) * 1e3 / args.launches)
            row = {"rows": lq, "keys": lk}
            row.update({f"{name}_us": round(float(np.median(t)), 2) for name, t in times.items()})
            row["weights_bytes"] = lq * lk * 4
            res.append(row)
            del graphs
    return res


def track_part(args, dev):
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, vanilla_args
    from trackformer_b200.tracker import Tracker

    cfg = dict(public_detections=False, detection_obj_score_thresh=0.5, track_obj_score_thresh=0.4,
               detection_nms_thresh=0.0, track_nms_thresh=0.0, steps_termination=1, prev_frame_dist=1,
               inactive_patience=-1, reid_sim_threshold=0.0, reid_sim_only=False, reid_score_thresh=0.4,
               reid_greedy_matching=False)
    arms = {}
    for maps in (False, True):
        for cls in (Tracker, DeviceTracker):
            torch.manual_seed(0)
            model, _, _ = build_model(vanilla_args(tracking=True, masks=True, dataset="mot", device=str(dev)))
            with torch.no_grad():
                model.class_embed.bias[0] += 8.0
            model.to(dev).tracking()
            tracker = cls(GraphedDetector(model, bucket=args.bucket), {"bbox": PostProcess()}, cfg, maps)
            tracker.reset()
            arms[f"{cls.__name__}_maps_{'on' if maps else 'off'}"] = tracker
    parts = {name: {"detect": [], "maps": []} for name in arms}

    def timed(name, part, fn):
        def call(*a, **kw):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **kw)
            torch.cuda.synchronize()
            parts[name][part].append((time.perf_counter() - t0) * 1e3)
            return r
        return call
    for name, tracker in arms.items():
        tracker._detect = timed(name, "detect", tracker._detect)
        tracker._attention_maps = timed(name, "maps", tracker._attention_maps)
    g = torch.Generator().manual_seed(1)
    frames = [torch.randn(1, 3, args.height, args.width, generator=g).pin_memory() for _ in range(4)]
    times = {name: [] for name in arms}
    nbytes = {name: [] for name in arms}
    for i in range(args.warmup + args.frames):
        for name, tracker in arms.items():
            for v in parts[name].values():
                v.append(None)                                # marks the start of this step's entries
            blob = {"img": frames[i % len(frames)], "orig_size": torch.tensor([[args.height, args.width]])}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tracker.step(blob)
            torch.cuda.synchronize()
            tracker.detection_obj_score_thresh = 2.0          # the first frame's tracks only: a steady track count
            if i >= args.warmup:
                times[name].append((time.perf_counter() - t0) * 1e3)
                fresh = int((np.asarray(tracker._result_rows) >= 0).sum()) if tracker.generate_attention_maps else 0
                hw = (-(-args.height // 32)) * (-(-args.width // 32))
                nbytes[name].append(fresh * hw * 4)
    def per_step(entries):
        """sum of each step's timed calls, steps after the warm-up"""
        steps, cur = [], None
        for e in entries:
            if e is None:
                if cur is not None:
                    steps.append(cur)
                cur = 0.0
            else:
                cur += e
        steps.append(cur)
        return steps[args.warmup:]
    out = {}
    for name in arms:
        det, maps = per_step(parts[name]["detect"]), per_step(parts[name]["maps"])
        rest = [t - d - m for t, d, m in zip(times[name], det, maps)]
        out[name + "_split"] = {"detect_ms_median": round(float(np.median(det)), 3),
                                "maps_ms_median": round(float(np.median(maps)), 3),
                                "rest_ms_median": round(float(np.median(rest)), 3)}
    for name in arms:
        out[name] = {"ms_per_step_median": round(float(np.median(times[name])), 3),
                     "ms_per_step_p90": round(float(np.percentile(times[name], 90)), 3),
                     "map_bytes_per_frame_mean": float(np.mean(nbytes[name])),
                     "tracks": len(arms[name].results)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="kernel,track")
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--height", type=int, default=800)
    ap.add_argument("--width", type=int, default=1333)
    ap.add_argument("--bucket", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attn_map_bench.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    name, limit = card()
    res = {"card": name, "power_limit": limit}
    parts = args.parts.split(",")
    if "kernel" in parts:
        res["kernel"] = kernel_part(args, dev)
    if "track" in parts:
        res["track"] = track_part(args, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
