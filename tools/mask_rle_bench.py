#!/usr/bin/env python
"""Kernel time of the MOTS run-length encoder (csrc/mask_rle.cu, `tfb200_mask_rle_i32`) on one GPU.

Label maps of the tracker's sizes (800x1333, the detector's input; 1080x1920, a MOTS20 frame) with `--tracks` ids
(default 100), of two kinds:
  * "boxes": person-like rectangles (a tenth to a half of the height, up to a twelfth of the width), later ones on top
    -- the few long runs per column of real masks;
  * "resolved": `resolve_track_masks` (csrc/track_masks.cu) of random stride-4 logits -- many short runs, the busy end
    of what the tracker produces.
Each shape's call is captured `--per-graph` times in one CUDA graph; a window replays it `--replays` times between two
CUDA events, the windows of all maps alternate, and the median window gives the time per call.  The strings are
checked against trackformer_b200.mots.encode first.  Prints one JSON line with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def boxes_map(H, W, T, seed):
    rng = np.random.default_rng(seed)
    lab = np.full((H, W), -1, np.int32)
    for i in range(T):
        h, w = int(rng.integers(H // 10, H // 2)), int(rng.integers(W // 40, W // 12))
        y, x = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
        lab[y:y + h, x:x + w] = i
    return torch.from_numpy(lab)


def resolved_map(H, W, T, seed, dev):
    from trackformer_b200.segmentation import resolve_track_masks
    g = torch.Generator().manual_seed(seed)
    size = ((H + 3) // 4 * 4, (W + 3) // 4 * 4)
    logits = (torch.randn(T, size[0] // 4, size[1] // 4, generator=g) * 4).to(dev)
    return resolve_track_masks(logits, list(range(T)), list(range(T)), None, size, size, (H, W)).cpu()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (v.strip() for v in out.split(","))
        return name, power
    except Exception as e:                                  # the numbers still stand with the torch device name
        return torch.cuda.get_device_name(0), f"not read ({type(e).__name__})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=100)
    ap.add_argument("--per-graph", type=int, default=20)
    ap.add_argument("--replays", type=int, default=10)
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    from trackformer_b200 import ext
    from trackformer_b200.mots import encode, label_map_rle
    assert torch.cuda.is_available(), "mask_rle_bench needs a CUDA device"
    dev = torch.device("cuda:0")
    ext.load()
    lib = ctypes.CDLL(ext.library_path())
    lib.tfb200_mask_rle_workspace_bytes.restype = ctypes.c_size_t
    lib.tfb200_mask_rle_workspace_bytes.argtypes = [ctypes.c_int] * 3
    lib.tfb200_mask_rle_max_bytes.restype = ctypes.c_int64
    lib.tfb200_mask_rle_max_bytes.argtypes = [ctypes.c_int] * 3
    f = lib.tfb200_mask_rle_i32
    f.restype = ctypes.c_int
    f.argtypes = ([ctypes.c_void_p] * 2 + [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                                                  ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p])
    T = args.tracks
    cases = []
    for H, W in ((800, 1333), (1080, 1920)):
        for kind in ("boxes", "resolved"):
            host = boxes_map(H, W, T, H) if kind == "boxes" else resolved_map(H, W, T, H, dev)
            lab = host.to(dev)
            ids = torch.arange(T, dtype=torch.int32, device=dev)
            rles = label_map_rle(lab, ids.cpu().numpy())
            flat = np.ascontiguousarray(host.numpy().T)
            assert all(r == encode((flat == t).T) for t, r in enumerate(rles)), (H, W, kind)
            ws_bytes = lib.tfb200_mask_rle_workspace_bytes(H, W, T)
            cap = lib.tfb200_mask_rle_max_bytes(H, W, T)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            chars = torch.empty(cap, dtype=torch.uint8, device=dev)
            header = torch.empty(2 + 2 * T, dtype=torch.int64, device=dev)

            def call():
                rc = f(lab.data_ptr(), ids.data_ptr(), H, W, T, ws.data_ptr(), ws_bytes, header.data_ptr(),
                       chars.data_ptr(), cap, torch.cuda.current_stream().cuda_stream)
                assert rc == 0, rc
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                call()                                      # warm-up outside the capture
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(args.per_graph):
                    call()
            graph.replay()
            torch.cuda.synchronize()
            h = header.cpu().numpy()
            assert h[0] == 0 and h[1] == sum(len(r["counts"]) for r in rles)
            cases.append({"H": H, "W": W, "kind": kind, "graph": graph, "buffers": (lab, ids, ws, chars, header),
                          "times": [], "string_bytes": int(h[1]),
                          "foreground": float((host >= 0).float().mean()), "label_bytes": H * W * 4})
    for _ in range(args.windows):                           # windows of all maps alternate
        for c in cases:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.replays):
                c["graph"].replay()
            b.record()
            b.synchronize()
            c["times"].append(a.elapsed_time(b) * 1e3 / (args.replays * args.per_graph))
    name, power = card()
    line = {"what": "tfb200_mask_rle_i32 kernel time per call (9 launches + 4 memsets), CUDA-graph replay",
            "card": name, "power_limit": power, "tracks": T, "per_graph": args.per_graph, "replays": args.replays,
            "windows": args.windows, "cases": []}
    for c in cases:
        t = np.asarray(c["times"])
        line["cases"].append({"shape": f"{c['H']}x{c['W']}", "kind": c["kind"], "us_median": float(np.median(t)),
                              "us_min": float(t.min()), "us_max": float(t.max()), "string_bytes": c["string_bytes"],
                              "label_bytes": c["label_bytes"], "foreground_share": round(c["foreground"], 4)})
    print(json.dumps(line))


if __name__ == "__main__":
    main()
