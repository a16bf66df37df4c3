#!/usr/bin/env python
"""Scoring tracking runs on the GPU (`trackformer_b200.mot_eval`) at the size of the MOTChallenge train splits.

Workloads (synthetic, seeded, tests/mot_eval_fixtures.py): `mot17` -- 7 sequences with the MOT17 train split's frame
counts (5,316 frames) and 15-45 people per frame; `mot20` -- 4 sequences with the MOT20 train split's frame counts
(8,931 frames) and 60-150 people per frame, about 1.1 M ground-truth boxes.  Hypotheses: the ground truth with
jitter, drops, id swaps and restarts, near-duplicates and false positives.

Per workload: the packing time (`get_mot_accum` over every sequence, host), the time of `evaluate_mot_accums` as a host
clock around work that ends in the read-back's synchronise (packing of the batch, one upload, the launches, one
read-back, the DataFrame), the CUDA-event time of the C entry's launches alone, the box pairs evaluated and found
valid, the largest residual and identity components met.  `--oracle` also times tests/mot_eval_reference.py -- the
Python / scipy restatement the tests compare against, not motmetrics -- on the same data, on the host, once, and
checks that its metrics equal the GPU's.  The card's name and power limit are read in the same run.  Prints one
JSON line.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOADS = {
    "mot17": [("MOT17-02", 600, 30), ("MOT17-04", 1050, 45), ("MOT17-05", 837, 15), ("MOT17-09", 525, 20),
              ("MOT17-10", 654, 25), ("MOT17-11", 900, 20), ("MOT17-13", 750, 15)],
    "mot20": [("MOT20-01", 429, 60), ("MOT20-02", 2782, 130), ("MOT20-03", 2405, 100), ("MOT20-05", 3315, 150)],
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                        text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def kernel_ms(accums, repeats):
    """CUDA-event time of tfb200_mot_eval_f32's launches alone (buffers uploaded and allocated beforehand)."""
    from trackformer_b200 import mot_eval
    buf, offsets, z = mot_eval._pack(accums)
    dev = torch.device("cuda")
    buf_dev = torch.from_numpy(buf).to(dev)
    out0, _ = mot_eval.evaluate_counters(accums)
    cap = int(out0[:, 1].sum())
    lib = mot_eval._library()
    ws_bytes = lib.tfb200_mot_eval_workspace_bytes(z["S"], z["F"], z["n_gt"], z["n_trk"], z["tp_cells"],
                                                   z["max_obj"], z["max_hyp"], cap)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(z["S"] * 16, dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    ptrs = [buf_dev.data_ptr() + o for o in offsets]
    times = []
    for _ in range(repeats + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rc = lib.tfb200_mot_eval_f32(*ptrs, z["S"], z["F"], z["n_gt"], z["n_trk"], z["tp_cells"], z["max_obj"],
                                     z["max_hyp"], cap, ws.data_ptr(), ws_bytes, out.data_ptr(), stream)
        b.record()
        assert rc == 0
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    assert (out.view(z["S"], 16).cpu().numpy() == out0).all()
    return float(np.median(times[1:])), out0, z, ws_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="mot17,mot20")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--oracle", action="store_true", help="also time the Python oracle once per workload")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mot_eval_bench needs a CUDA device"
    import mot_eval_fixtures as mf
    from trackformer_b200 import mot_eval
    name, power = card()
    report = {"card": name, "power_limit": power, "workloads": {}}
    for wl in args.workloads.split(","):
        seqs = WORKLOADS[wl]
        data = {n: mf.scene(i + (0 if wl == "mot17" else 50), n_frames=f, n_objects=k, size=(45.0, 110.0),
                            fp_rate=2.0, p_swap=0.0005, p_restart=0.002)
                for i, (n, f, k) in enumerate(seqs)}
        t0 = time.perf_counter()
        accums = [mot_eval.get_mot_accum(r, fr) for r, fr in data.values()]
        pack_s = time.perf_counter() - t0
        names = list(data)
        mot_eval.evaluate_mot_accums(accums, names)                 # warm-up: module load, allocator
        walls = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            summary, text = mot_eval.evaluate_mot_accums(accums, names)
            walls.append(time.perf_counter() - t0)
        k_ms, out, z, ws_bytes = kernel_ms(accums, args.repeats)
        r = {"sequences": len(seqs), "frames": z["F"], "gt_boxes": z["n_obj"], "track_boxes": z["n_hyp"],
             "gt_ids": z["n_gt"], "track_ids": z["n_trk"], "pairs_evaluated": z["products"],
             "valid_pairs": int(out[:, 1].sum()), "largest_residual_component": [int(out[:, 11].max()),
                                                                                  int(out[:, 12].max())],
             "largest_identity_component": [int(out[:, 13].max()), int(out[:, 14].max())],
             "workspace_mb": round(ws_bytes / 2 ** 20, 1), "get_mot_accum_s": round(pack_s, 3),
             "evaluate_ms_median": round(1e3 * float(np.median(walls)), 2),
             "evaluate_ms_min": round(1e3 * min(walls), 2), "kernels_ms_median": round(k_ms, 2),
             "mota": float(summary["mota"]["OVERALL"]), "idf1": float(summary["idf1"]["OVERALL"])}
        if args.oracle:
            import mot_eval_reference as ref
            t0 = time.perf_counter()
            expected = ref.evaluate({n: ref.counts(ref.accumulate(res, [f["gt"] for f in fr]))
                                     for n, (res, fr) in data.items()})
            r["oracle_cpu_s"] = round(time.perf_counter() - t0, 2)
            for n in expected:
                for col in mot_eval.COLUMNS:
                    want, got = float(expected[n][col]), float(summary[col][n])
                    assert abs(want - got) <= 1e-12 or (np.isnan(want) and np.isnan(got)), (wl, n, col, got, want)
            r["oracle_equal"] = True
        else:
            r["oracle_cpu_s"] = "not measured"
        print(text, file=sys.stderr)
        report["workloads"][wl] = r
    print(json.dumps(report))


if __name__ == "__main__":
    main()
