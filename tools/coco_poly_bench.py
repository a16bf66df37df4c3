"""Time polygon ground-truth rasterisation on the GPU (trackformer_b200.coco_masks, csrc/coco_poly.cu).

  (a) `coco_eval.GroundTruth(dataset, True, device=)` for a synthetic COCO-val-sized set: 5,000 images, about 36,000
      polygon annotations of 1 - 4 parts of 8 - 80 vertices (tests/coco_poly_fixtures.py coco_val_like, seed 0);
      also `coco_masks.poly_runs` alone (pack, upload, both calls and the read-backs)
  (b) `convert_coco_poly_to_mask` for one 480 x 640 image with 7 instances

Each GPU time is the median of --repeats runs that end in a device synchronise, after a warm-up.  With --oracle the
same inputs also go through the g++ build of the kernels' source (tests/host_build/coco_poly_host.cpp, the whole set,
compiled to a temporary directory) and the plain-Python restatement of pycocotools (tests/coco_poly_reference.py, the
first --oracle-anns annotations of (a), and all of (b)).  pycocotools is not a dependency and is not measured.
Prints one JSON line with the card's name and power limit, read in the same run.

  python tools/coco_poly_bench.py [--oracle] [--repeats 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import coco_poly_fixtures as pf  # noqa: E402
from trackformer_b200 import coco_eval, coco_masks  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, repeats, dev):
    fn()
    torch.cuda.synchronize(dev)
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize(dev)
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def host_build_seconds(segs, hw):
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libcoco_poly_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared",
                               os.path.join(ROOT, "tests", "host_build", "coco_poly_host.cpp"), "-o", so])
        lib = ctypes.CDLL(so)
        names = [str(i) for i in range(len(segs))]
        t0 = time.perf_counter()
        z = coco_masks.pack_polygons(segs, hw, names)
        P, A, E = coco_masks.geometry(z)
        geo = [z[k].ctypes.data for k in ("xy", "part_off", "part_ann", "ann_part", "ann_hw")] + [P, A, E]
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
        lib.tfb200_coco_poly_count_host.argtypes = [vp] * 5 + [i32, i32, i64, vp, vp, vp]
        lib.tfb200_coco_poly_runs_host.argtypes = [vp] * 5 + [i32, i32, i64, vp, i64, vp, vp]
        toggle_off, ann_points = np.zeros(E + 1, np.int32), np.zeros(max(A, 1), np.int64)
        sizes = np.zeros(coco_masks.SIZES, np.int64)
        lib.tfb200_coco_poly_count_host(*geo, toggle_off.ctypes.data, ann_points.ctypes.data, sizes.ctypes.data)
        run_off, runs = np.zeros(A + 1, np.int64), np.zeros((max(int(sizes[1]), 1), 2), np.uint32)
        lib.tfb200_coco_poly_runs_host(*geo, toggle_off.ctypes.data, int(sizes[1]), run_off.ctypes.data,
                                       runs.ctypes.data)
        return time.perf_counter() - t0, sizes, run_off, runs[:run_off[-1]].astype(np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--oracle-anns", type=int, default=300)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("coco_poly_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {"card": card(), "torch_device": torch.cuda.get_device_name(dev)}

    ds = pf.coco_val_like(0)
    anns = ds["annotations"]
    hw = [(ds["images"][a["image_id"] - 1]["height"], ds["images"][a["image_id"] - 1]["width"]) for a in anns]
    segs = [a["segmentation"] for a in anns]
    names = [str(a["id"]) for a in anns]
    out["a_images"], out["a_annotations"] = len(ds["images"]), len(anns)
    out["a_parts"] = sum(len(s) for s in segs)
    out["a_ground_truth_s"] = timed(lambda: coco_eval.GroundTruth(ds, True, dev), args.repeats, dev)
    out["a_poly_runs_s"] = timed(lambda: coco_masks.poly_runs(segs, hw, names, dev), args.repeats, dev)
    off, runs = coco_masks.poly_runs(segs, hw, names, dev)
    out["a_runs"] = int(off[-1])

    rng = np.random.default_rng(1)
    inst = [pf.segmentation(rng, 480, 640) for _ in range(7)]
    out["b_convert_s"] = timed(lambda: coco_masks.convert_coco_poly_to_mask(inst, 480, 640, dev), 10 * args.repeats,
                               dev)

    if args.oracle:
        import coco_poly_reference as ref
        t, sizes, h_off, h_runs = host_build_seconds(segs, hw)
        out["a_boundary_points"], out["a_toggles"] = int(sizes[0]), int(sizes[1])
        out["a_host_build_s"] = t
        out["a_host_build_equal"] = bool(np.array_equal(h_off, off) and np.array_equal(h_runs, runs))
        n = min(args.oracle_anns, len(anns))
        t0 = time.perf_counter()
        got = [ref.ann_runs(segs[i], *hw[i]) for i in range(n)]
        out["a_python_oracle_s_first_anns"], out["a_python_oracle_anns"] = time.perf_counter() - t0, n
        out["a_python_oracle_equal"] = all(np.array_equal(g, runs[off[i]:off[i + 1]]) for i, g in enumerate(got))
        t0 = time.perf_counter()
        want = np.stack([ref.ann_mask(s, 480, 640) for s in inst])
        out["b_python_oracle_s"] = time.perf_counter() - t0
        out["b_equal"] = bool(torch.equal(coco_masks.convert_coco_poly_to_mask(inst, 480, 640, dev).cpu(),
                                          torch.from_numpy(want)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
