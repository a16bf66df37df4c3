"""Time panoptic post-processing (`PostProcessPanoptic`, csrc/panoptic.cu) and PQ scoring (`PanopticEvaluator`,
`pq_compute`) on an H100.

  post   batch 2, 100 queries, 251 class logits, stride-4 masks of an 800 x 1216 padded batch (200 x 304), processed at
         800 x 1066 and 790 x 1050, resized to 480 x 640.  Arms, alternated over --windows: the kernels with the maps
         left on the device (`label_maps`), the kernels plus the host PNG encode (`forward`), and the reference's
         composition on the same GPU (the tests' torch restatement, tests/panoptic_restatement.py); the PNG encode of
         one batch is also timed alone.
  pq     a synthetic COCO-panoptic-val-sized workload: --images (5,000) images of 480 x 640, 133 categories (80
         things), ~11 GT and ~20 predicted rectangle segments per image: `update` per batch of 2 from device maps,
         `summarize`, the whole evaluation from device maps and `pq_compute` from PNG folders; with --oracle the numpy
         oracle (tests/panoptic_eval_reference.py) timed once and its result checked equal.  panopticapi itself is not
         installed and is not measured.

Each time ends in a device synchronise; medians with p10 / p90 over the windows.  Prints one JSON line per part with
the card's name and power limit.  Scratch files go to a temporary directory.  Stops without a CUDA device.

  python tools/panoptic_bench.py [--parts post,pq] [--images 5000] [--oracle]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from trackformer_b200 import panoptic_eval as pe  # noqa: E402
from trackformer_b200.segmentation import PostProcessPanoptic  # noqa: E402

IS_THING = {i: i <= 90 for i in range(201)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def stats(xs):
    xs = np.asarray(xs) * 1e3
    return {"median_ms": float(np.median(xs)), "p10_ms": float(np.percentile(xs, 10)),
            "p90_ms": float(np.percentile(xs, 90))}


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, r


def bench_post(windows):
    import panoptic_restatement as rs
    g = torch.Generator().manual_seed(0)
    B, Q = 2, 100
    logits = torch.randn(B, Q, 251, generator=g)
    for b in range(B):
        q = torch.randperm(Q, generator=g)[:30]
        logits[b, q, torch.randint(1, 201, (30,), generator=g)] += 12.0
    outputs = {"pred_logits": logits.cuda(), "pred_masks": (torch.randn(B, Q, 200, 304, generator=g) * 3).cuda()}
    sizes, tsizes = [(800, 1066), (790, 1050)], [(480, 640), (480, 640)]
    post = PostProcessPanoptic(IS_THING)
    arms = {"kernels_device_maps": lambda: post.label_maps(outputs, sizes, tsizes),
            "kernels_png": lambda: post(outputs, sizes, tsizes),
            "reference_composition": lambda: rs.postprocess(outputs, sizes, tsizes, IS_THING)}
    for f in arms.values():
        f()
    times = {k: [] for k in arms}
    for _ in range(windows):
        for k, f in arms.items():
            times[k].append(timed(f)[0])
    maps, _ = post.label_maps(outputs, sizes, tsizes)
    host = [m.cpu().numpy() for m in maps]
    enc = []
    for _ in range(windows):
        t = time.perf_counter()
        for m in host:
            pe.png_of(m)
        enc.append(time.perf_counter() - t)
    res = {k: stats(v) for k, v in times.items()}
    res["png_encode_batch"] = stats(enc)
    return res


def pq_workload(n_images, seed=0, H=480, W=640):
    rng = np.random.default_rng(seed)
    cats = [{"id": c, "isthing": int(k < 80), "name": str(c)} for k, c in enumerate(range(1, 134))]
    gt_anns, pred_anns, gmaps, pmaps = [], [], {}, {}
    for i in range(n_images):
        gm = np.zeros((H, W), np.int32)
        segs = []
        for s in range(int(rng.poisson(11)) + 1):
            y0, x0 = rng.integers(0, H - 20), rng.integers(0, W - 20)
            gm[y0:y0 + rng.integers(20, H // 2), x0:x0 + rng.integers(20, W // 2)] = 1 + s * 7919
        ids, cnt = np.unique(gm, return_counts=True)
        for gid, a in zip(ids.tolist(), cnt.tolist()):
            if gid:
                segs.append({"id": gid, "category_id": int(rng.integers(1, 134)), "area": a,
                             "iscrowd": int(rng.random() < 0.05)})
        pm = np.zeros((H, W), np.int32)
        psegs = []
        for s in range(int(rng.poisson(20)) + 1):
            if segs and rng.random() < 0.6:
                src = segs[rng.integers(len(segs))]
                ys, xs = np.nonzero(gm == src["id"])
                dy, dx = rng.integers(-8, 9, 2)
                pm[max(0, ys.min() + dy):ys.max() + dy, max(0, xs.min() + dx):xs.max() + dx] = s
                psegs.append({"id": s, "category_id": src["category_id"]})
            else:
                y0, x0 = rng.integers(0, H - 10), rng.integers(0, W - 10)
                pm[y0:y0 + rng.integers(10, H // 4), x0:x0 + rng.integers(10, W // 4)] = s
                psegs.append({"id": s, "category_id": int(rng.integers(1, 134))})
        present = set(np.unique(pm).tolist())
        psegs = [p for p in psegs if p["id"] in present]
        fname = f"{i:012d}.png"
        gt_anns.append({"image_id": i, "file_name": fname, "segments_info": segs})
        pred_anns.append({"image_id": i, "file_name": fname, "segments_info": psegs})
        gmaps[i], pmaps[i] = gm, pm
        if (i + 1) % 500 == 0:
            print(f"[panoptic_bench] {i + 1} of {n_images} images generated", file=sys.stderr, flush=True)
    return {"categories": cats, "annotations": gt_anns}, {"annotations": pred_anns}, gmaps, pmaps


def bench_pq(n_images, oracle, tmp):
    gt_json, pred_json, gmaps, pmaps = pq_workload(n_images)
    for side, js, maps in (("gt", gt_json, gmaps), ("pred", pred_json, pmaps)):
        os.makedirs(os.path.join(tmp, side))
        for a in js["annotations"]:
            Image.fromarray(pe.id2rgb(maps[a["image_id"]])).save(os.path.join(tmp, side, a["file_name"]))
        print(f"[panoptic_bench] {side} PNG folder written", file=sys.stderr, flush=True)
        with open(os.path.join(tmp, side + ".json"), "w") as f:
            json.dump(js, f)
    pngs = {a["image_id"]: pe.png_of(pmaps[a["image_id"]]) for a in pred_json["annotations"][:2]}
    dev_maps = {i: torch.from_numpy(m).cuda() for i, m in pmaps.items()}
    res = {"images": n_images, "gt_segments": sum(len(a["segments_info"]) for a in gt_json["annotations"]),
           "pred_segments": sum(len(a["segments_info"]) for a in pred_json["annotations"])}

    def evaluate():
        ev = pe.PanopticEvaluator(os.path.join(tmp, "gt.json"), os.path.join(tmp, "gt"), os.path.join(tmp, "out"))
        upd = []
        anns = pred_json["annotations"]
        for c in range(0, len(anns), 2):
            preds = [dict(a, png_string=pngs.get(a["image_id"], b""), label_map=dev_maps[a["image_id"]])
                     for a in anns[c:c + 2]]
            upd.append(timed(lambda: ev.update(preds))[0])
        t, r = timed(ev.summarize)
        return upd, t, r
    evaluate()                                             # warm-up (module load, allocator)
    print("[panoptic_bench] warm-up evaluation done", file=sys.stderr, flush=True)
    t_all, (upd, t_sum, got) = timed(evaluate)
    res["update_per_batch2"] = stats(upd)
    res["summarize_ms"] = t_sum * 1e3
    res["evaluate_device_maps_s"] = t_all
    t_png, got_png = timed(lambda: pe.pq_compute(os.path.join(tmp, "gt.json"), os.path.join(tmp, "pred.json"),
                                                 os.path.join(tmp, "gt"), os.path.join(tmp, "pred")))
    res["pq_compute_png_folders_s"] = t_png
    res["device_maps_equal_png_folders"] = got == got_png
    res["PQ_all"] = got["All"]
    if oracle:
        import panoptic_eval_reference as ref
        t = time.perf_counter()
        want = ref.pq_compute(gt_json, pred_json, gmaps, pmaps)[0]
        res["oracle_s"] = time.perf_counter() - t
        res["oracle_max_abs_diff"] = max(abs(got[n][k] - want[n][k]) for n in ("All", "Things", "Stuff")
                                         for k in ("pq", "sq", "rq"))
        res["oracle_equal_1e-12"] = res["oracle_max_abs_diff"] <= 1e-12 and all(
            got[n]["n"] == want[n]["n"] for n in ("All", "Things", "Stuff"))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="post,pq")
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--windows", type=int, default=20)
    ap.add_argument("--oracle", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("panoptic_bench needs a CUDA device")
    gpu = card()
    parts = args.parts.split(",")
    if "post" in parts:
        print(json.dumps({"part": "post", "card": gpu, **bench_post(args.windows)}), flush=True)
    if "pq" in parts:
        with tempfile.TemporaryDirectory() as tmp:
            print(json.dumps({"part": "pq", "card": gpu, **bench_pq(args.images, args.oracle, tmp)}), flush=True)


if __name__ == "__main__":
    main()
