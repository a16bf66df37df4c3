#!/usr/bin/env python
"""Frame ingest on one GPU: the resize + normalise kernel alone, and online tracking fed raw uint8 frames against
tracking fed pre-processed float images.  Prints one JSON line with the card name and power limit (query only), and
writes it to --out when given.

--parts kernel  csrc/frame_ingest.cu through FrameIngest on device-resident uint8 frames (eight different frames in
                rotation), CUDA-event medians over windows alternated between the shapes:
                  1080x1920 -> 750x1333    both passes (ksize 5)
                  800x1333  -> 800x1333    both passes skipped: table look-up and layout change only
                  480x640   -> 800x1066    enlargement (ksize 3)
                with the bytes the kernel has to move (uint8 frame in, fp32 planes out; the coefficient tables are a
                few tens of KB) computed from the shapes, the resulting GB/s and its share of 3.35 TB/s.
--parts track   DeviceTracker.step over GraphedDetector (deformable tracking model, random weights with one confident
                class) on a 1080x1920 synthetic video, three arms alternated frame by frame, each with its own tracker:
                  frame         blob["frame"]: pageable host uint8 -> pinned staging -> device -> kernel -> step
                  img           blob["img"]: the pre-made 750x1333 float image in pinned host memory -> step
                  host_pre+img  the reference-shaped host work per frame (Pillow bilinear resize + to_tensor + normalize
                                on one thread; torch's antialiased F.interpolate on the CPU where Pillow is missing --
                                "host_reference" says which), then blob["img"] from the pageable result
                Host milliseconds of the pre-processing are reported separately from the step.

Needs a CUDA device: without one it stops after checking its arguments and the host reference, it never falls back.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12                              # H100 SXM data sheet
KERNEL_SHAPES = {"1080x1920": (1080, 1920), "800x1333": (800, 1333), "480x640": (480, 640)}
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:                                   # noqa: BLE001  (no nvidia-smi: the limit stays unknown)
        return torch.cuda.get_device_name(0), "unknown"


def kernel_bytes(shape, size):
    """bytes one call has to move: the interleaved uint8 frame in, three fp32 planes out"""
    return shape[0] * shape[1] * 3 + size[0] * size[1] * 3 * 4


def host_reference():
    """(name, fn): fn(uint8 [H, W, 3] array, (h, w)) -> fp32 [1, 3, h, w] the way the reference's datasets make it"""
    try:
        from PIL import Image
        import torchvision.transforms.functional as F

        def pillow(frame, size):
            img = Image.fromarray(frame).resize((size[1], size[0]), Image.BILINEAR)
            return F.normalize(F.to_tensor(img), MEAN, STD)[None]
        return "pillow", pillow
    except ImportError:
        mean, std = torch.tensor(MEAN).view(1, 3, 1, 1), torch.tensor(STD).view(1, 3, 1, 1)

        def interpolate(frame, size):
            x = torch.from_numpy(frame).permute(2, 0, 1)[None].float()
            x = torch.nn.functional.interpolate(x, size=size, mode="bilinear", antialias=True, align_corners=False)
            return x.div(255).sub(mean).div(std)
        return "F.interpolate(antialias=True) on the CPU (Pillow missing: not the reference's bytes)", interpolate


def video(shape, n, seed=2):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, shape + (3,)).astype(np.float32)
    return [np.clip(base + 4.0 * rng.standard_normal(shape + (3,)).astype(np.float32), 0, 255).astype(np.uint8)
            for _ in range(n)]


def stats(v):
    return {"median": statistics.median(v), "p10": float(np.percentile(v, 10)), "p90": float(np.percentile(v, 90))}


def bench_kernel(args, dev, result):
    from trackformer_b200.frame_ingest import FrameIngest
    ingest = FrameIngest(dev)
    frames = {k: [torch.from_numpy(f).to(dev) for f in video(s, 8, seed=i)] for i, (k, s) in enumerate(KERNEL_SHAPES.items())}
    times = {k: [] for k in frames}
    for k in frames:                                    # tables, buffers, module load
        for f in frames[k]:
            ingest(f)
    torch.cuda.synchronize()
    graphs = {}
    for k, fs in frames.items():                        # one graph of `iters` launches per shape: the kernel takes a few
        graphs[k] = torch.cuda.CUDAGraph()              # microseconds, less than it costs to launch it from Python
        with torch.cuda.graph(graphs[k]):
            for i in range(args.iters):
                ingest(fs[i % len(fs)])
        graphs[k].replay()
    torch.cuda.synchronize()
    for _ in range(args.repeats):
        for k in frames:
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            graphs[k].replay()
            stop.record()
            stop.synchronize()
            times[k].append(start.elapsed_time(stop) / args.iters)
    rows = {}
    for k, shape in KERNEL_SHAPES.items():
        size = result["sizes"][k]
        ms, nbytes = statistics.median(times[k]), kernel_bytes(shape, size)
        rows[k] = {"to": "x".join(map(str, size)), "ms": ms, "ms_min": min(times[k]), "ms_max": max(times[k]),
                   "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6, "share_of_3.35TBps": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
    result["kernel"] = {"iters": args.iters, "windows": args.repeats, "rows": rows}
    print("kernel", json.dumps(result["kernel"]), flush=True)


def bench_track(args, dev, result, host_fn):
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.frame_ingest import FrameIngest, val_size
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args
    shape = (1080, 1920)
    size = val_size(*shape)
    torch.manual_seed(0)
    model, _, _ = build_model(default_args(True, False, device=str(dev)))
    with torch.no_grad():
        for name, p in model.named_parameters():       # random weights: make class 0 confident so tracks exist
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 6.0
    model.to(dev).eval()
    model.tracking()
    cfg = dict(public_detections=False, detection_obj_score_thresh=0.4, track_obj_score_thresh=0.4,
               detection_nms_thresh=0.9, track_nms_thresh=0.9, steps_termination=1, prev_frame_dist=1,
               inactive_patience=-1, reid_sim_threshold=0.0, reid_sim_only=False, reid_score_thresh=0.4,
               reid_greedy_matching=False)
    frames = video(shape, 4)
    ingest = FrameIngest(dev)
    pinned = [ingest(f)["img"].cpu().pin_memory() for f in frames]
    orig, dets = torch.tensor([list(shape)]), torch.zeros(1, 0, 4)

    def blob_frame(i):
        return {"frame": frames[i % 4], "dets": dets}, 0.0

    def blob_img(i):
        return {"img": pinned[i % 4], "orig_size": orig, "dets": dets}, 0.0

    def blob_host(i):
        t0 = time.perf_counter()
        img = host_fn(frames[i % 4], size)
        return {"img": img, "orig_size": orig, "dets": dets}, (time.perf_counter() - t0) * 1e3
    arms = {"frame": blob_frame, "img": blob_img, "host_pre+img": blob_host}
    trackers = {}
    for a in arms:
        trackers[a] = DeviceTracker(GraphedDetector(model), {"bbox": DeformablePostProcess()}, cfg, False,
                                    frame_ingest=FrameIngest(dev))
        trackers[a].reset()
    step_ms, pre_ms = {a: [] for a in arms}, {a: [] for a in arms}
    with torch.no_grad():
        for i in range(args.warmup + args.frames):
            for a, make in arms.items():
                blob, pre = make(i)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                trackers[a].step(blob)
                torch.cuda.synchronize()
                if i >= args.warmup:
                    step_ms[a].append((time.perf_counter() - t0) * 1e3)
                    pre_ms[a].append(pre)
    ids = {a: sorted(trackers[a].get_results()) for a in arms}
    float_bytes, frame_bytes = size[0] * size[1] * 3 * 4, shape[0] * shape[1] * 3
    result["track"] = {
        "workload": f"DeviceTracker.step over GraphedDetector, deformable tracking model, {shape[0]}x{shape[1]} uint8 "
                    f"frames -> {size[0]}x{size[1]}", "frames": args.frames, "warmup": args.warmup,
        "step_ms": {a: stats(step_ms[a]) for a in arms},
        "host_preprocess_ms": {a: stats(pre_ms[a]) for a in arms},
        "h2d_image_bytes_per_frame": {"frame": frame_bytes, "img": float_bytes, "host_pre+img": float_bytes},
        "tracks": {a: len(ids[a]) for a in arms},
        "same_track_ids_frame_vs_img": ids["frame"] == ids["img"],
        "graph_captures": {a: trackers[a].obj_detector.captures for a in arms},
    }
    print("track", json.dumps(result["track"]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="kernel,track")
    ap.add_argument("--iters", type=int, default=200, help="kernel calls per timed window")
    ap.add_argument("--repeats", type=int, default=7, help="windows per shape, alternated")
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    parts = args.parts.split(",")
    unknown = sorted(set(parts) - {"kernel", "track"})
    if unknown or args.iters < 1 or args.repeats < 1 or args.frames < 1 or args.warmup < 0:
        ap.error(f"unknown parts {unknown}" if unknown else "--iters, --repeats, --frames must be >= 1, --warmup >= 0")
    from trackformer_b200.frame_ingest import val_size
    name, host_fn = host_reference()
    probe = host_fn(video((120, 160), 1)[0], (96, 128))
    assert probe.dtype == torch.float32 and tuple(probe.shape) == (1, 3, 96, 128)
    result = {"host_reference": name, "sizes": {k: list(val_size(*s)) for k, s in KERNEL_SHAPES.items()},
              "kernel_bytes": {k: kernel_bytes(s, val_size(*s)) for k, s in KERNEL_SHAPES.items()}}
    if not torch.cuda.is_available():
        print(json.dumps(result))
        sys.exit("ingest_bench needs a CUDA device: nothing was measured")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    result["gpu"], result["power_limit"] = card()
    if "kernel" in parts:
        bench_kernel(args, dev, result)
    if "track" in parts:
        bench_track(args, dev, result, host_fn)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
