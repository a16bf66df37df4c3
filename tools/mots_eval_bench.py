#!/usr/bin/env python
"""Scoring MOTS runs on the GPU (`trackformer_b200.mots_eval`) at the size of the MOTS20 train split.

Workload (synthetic, seeded, tests/mots_eval_fixtures.py `mots20_workload`): the size of MOTS20 train -- 4 sequences
of 600, 837, 525 and 900 frames, MOTS20-05 at 480 x 640 and the others at 1080 x 1920, 26,753 GT masks over 226 GT
tracks (11 slots per sequence, each a succession of people), an ignore region in half the frames, hypotheses with
jitter, misses, id switches, false positives and some inside the ignore region.  Two mask styles: `person` (one row
range per column) and `fragmented` (many short runs per column, several KB of string per mask).

Per style: `get_mots_accum` time over every sequence (host), the median host-clock time of `evaluate_mots_accums`
(packing, one upload, the launches, one read-back, the DataFrame), the CUDA-event time of the C entry alone, the
intervals, intersecting and valid pairs.  `--oracle` also runs tests/mots_eval_reference.py once (dense numpy masks
from `mots.decode`, the frames spread over a process pool of --processes workers, the matching in this process), reports
its wall time, and checks that its metrics equal the GPU's.  The card's name and power limit are read in the same run.
Prints one JSON line; stops without a CUDA device.
"""
import argparse
import json
import multiprocessing
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                        text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def kernel_ms(accums, repeats):
    """CUDA-event time of tfb200_mots_eval's launches alone (buffers uploaded and allocated beforehand)."""
    from trackformer_b200 import mots_eval
    buf, offsets, z = mots_eval._pack(accums)
    dev = torch.device("cuda")
    buf_dev = torch.from_numpy(buf).to(dev)
    lib = mots_eval._library()
    args = mots_eval._entry_args(z)
    ws_bytes = lib.tfb200_mots_eval_workspace_bytes(*args)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(z["S"] * (16 + mots_eval._XSLOTS), dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    ptrs = [buf_dev.data_ptr() + o for o in offsets]
    times, first = [], None
    for _ in range(repeats + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rc = lib.tfb200_mots_eval(*ptrs, *args, ws.data_ptr(), ws_bytes, out.data_ptr(), stream)
        b.record()
        assert rc == 0
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
        o = out.cpu().numpy()
        assert first is None or (o == first).all()
        first = o
    return float(np.median(times[1:])), mots_eval.check_counters(first, z), z, ws_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--styles", default="person,fragmented")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--oracle", action="store_true", help="also time the dense numpy oracle once per style")
    ap.add_argument("--processes", type=int, default=os.cpu_count(), help="workers building the data and the oracle")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mots_eval_bench needs a CUDA device"
    import mots_eval_fixtures as msf
    from trackformer_b200 import mots_eval
    name, power = card()
    report = {"card": name, "power_limit": power, "cpus": os.cpu_count(), "processes": args.processes, "styles": {}}
    pool = multiprocessing.get_context("spawn").Pool(args.processes)     # spawn: no fork of a CUDA process
    for style in args.styles.split(","):
        data = msf.mots20_workload(style, pool)
        t0 = time.perf_counter()
        accums = [mots_eval.get_mots_accum(*v) for v in data.values()]
        pack_s = time.perf_counter() - t0
        names = list(data)
        mots_eval.evaluate_mots_accums(accums, names)                 # warm-up: module load, allocator
        walls = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            summary, text = mots_eval.evaluate_mots_accums(accums, names)
            walls.append(time.perf_counter() - t0)
        k_ms, out, z, ws_bytes = kernel_ms(accums, args.repeats)
        x = out[:, 16:]
        r = {"sequences": len(accums), "frames": z["F"], "masks": z["n_masks"],
             "gt_masks": int(x[:, mots_eval._XGTDETS].sum()), "gt_tracks": z["n_gt"], "result_tracks": z["n_trk"],
             "string_mb": round(sum(len(a.chars) for a in accums) / 2 ** 20, 1),
             "intervals": int(x[:, mots_eval._XINTERVALS].sum()),
             "intersecting_pairs": int(x[:, mots_eval._XINTERSECTING].sum()), "valid_pairs": int(out[:, 1].sum()),
             "removed_hypotheses": int(x[:, mots_eval._XREMOVED].sum()), "workspace_mb": round(ws_bytes / 2 ** 20, 1),
             "get_mots_accum_s": round(pack_s, 3), "evaluate_ms_median": round(1e3 * float(np.median(walls)), 2),
             "evaluate_ms_min": round(1e3 * min(walls), 2), "kernels_ms_median": round(k_ms, 2),
             "smotsa": float(summary["smotsa"]["OVERALL"]), "idf1": float(summary["idf1"]["OVERALL"])}
        if args.oracle:
            import mots_eval_reference as ref
            t0 = time.perf_counter()
            expected = ref.evaluate({n: ref.counts(*ref.accumulate(*v, pool=pool)) for n, v in data.items()})
            r["oracle_wall_s"] = round(time.perf_counter() - t0, 2)
            for n in expected:
                for col in mots_eval.COLUMNS:
                    want, got = float(expected[n][col]), float(summary[col][n])
                    assert abs(want - got) <= 1e-12 or (np.isnan(want) and np.isnan(got)), (style, n, col, got, want)
            r["oracle_equal"] = True
        else:
            r["oracle_wall_s"] = "not measured"
        print(text, file=sys.stderr)
        report["styles"][style] = r
    pool.close()
    pool.join()
    print(json.dumps(report))


if __name__ == "__main__":
    main()
