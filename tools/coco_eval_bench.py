"""Time `trackformer_b200.coco_eval.CocoEvaluator` on synthetic workloads the size of the project's validation sets.

  mot17       2,650 frames, 1 category, ~30 GT boxes and 300 detections per frame (MOT17 half-split validation)
  crowdhuman  4,370 images, 1 category, ~23 people each
  coco        5,000 images, 80 categories, 100 detections each (COCO val2017)
  mots20      MOTS20 segm at 1080 x 1920, ~12 GT masks and 100 detections per frame (--frames, default 200)

Reports per workload the mean `update` time per batch (--batch images), the `accumulate` time and the whole
evaluation (updates + synchronize + accumulate), each ending in a device synchronise, and with --oracle the plain
Python oracle of tests/coco_eval_reference.py on the host, timed once.  pycocotools is not a dependency of the
project and is not measured.  Prints one JSON line per workload and the card's name and power limit.

  python tools/coco_eval_bench.py [--workloads mot17,crowdhuman,coco,mots20] [--oracle]
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
from trackformer_b200 import coco_eval as ce  # noqa: E402
from trackformer_b200 import mots  # noqa: E402


def boxes_workload(rng, n_img, n_cat, gt_per, det_per, h=1080, w=1920):
    images, anns, preds = [], [], {}
    for i in range(n_img):
        images.append({"id": i, "height": h, "width": w})
        n_gt = int(rng.poisson(gt_per))
        xy = rng.uniform(0, [w - 100, h - 200], (n_gt, 2))
        wh = rng.uniform([10, 20], [100, 200], (n_gt, 2))
        cats = rng.integers(1, n_cat + 1, n_gt)
        for g in range(n_gt):
            anns.append({"id": len(anns), "image_id": i, "category_id": int(cats[g]),
                         "bbox": [float(xy[g, 0]), float(xy[g, 1]), float(wh[g, 0]), float(wh[g, 1])],
                         "area": float(wh[g, 0] * wh[g, 1]), "iscrowd": int(rng.random() < 0.02)})
        src = rng.integers(0, max(n_gt, 1), det_per)
        jit = rng.normal(0, 4, (det_per, 4))
        b = np.zeros((det_per, 4), np.float32)
        if n_gt:
            b[:, :2] = xy[src] + jit[:, :2]
            b[:, 2:] = xy[src] + wh[src] + jit[:, 2:]
        fake = rng.random(det_per) < 0.5
        b[fake, :2] = rng.uniform(0, [w - 100, h - 200], (int(fake.sum()), 2))
        b[fake, 2:] = b[fake, :2] + rng.uniform(10, 150, (int(fake.sum()), 2))
        labels = (cats[src] - 1 if n_gt else rng.integers(0, n_cat, det_per)).astype(np.int64)
        preds[i] = {"scores": torch.from_numpy(rng.random(det_per).astype(np.float32)),
                    "labels": torch.from_numpy(labels), "boxes": torch.from_numpy(b)}
    return {"images": images, "annotations": anns, "categories": [{"id": c + 1} for c in range(n_cat)]}, preds


def mots_workload(rng, n_img, gt_per=12, det_per=100, h=1080, w=1920):
    images, anns, preds = [], [], {}
    for i in range(n_img):
        images.append({"id": i, "height": h, "width": w})
        ell = []
        for _ in range(gt_per):
            cx, cy = rng.uniform(100, w - 100), rng.uniform(150, h - 150)
            rx, ry = rng.uniform(15, 60), rng.uniform(40, 140)
            ell.append((cx, cy, rx, ry))
            y0, y1, x0, x1 = int(cy - ry), int(cy + ry) + 1, int(cx - rx), int(cx + rx) + 1
            yy, xx = np.mgrid[y0:y1, x0:x1]
            m = np.zeros((h, w), bool)
            m[y0:y1, x0:x1] = ((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 <= 1
            rle = mots.encode(m)
            rle["counts"] = rle["counts"].decode()
            anns.append({"id": len(anns) + 1, "image_id": i, "category_id": 1, "segmentation": rle,
                         "area": float(m.sum()), "iscrowd": 0, "bbox": [x0, y0, x1 - x0, y1 - y0]})
        preds[i] = dict(ell=ell, n=det_per, seed=int(rng.integers(1 << 30)))
    return {"images": images, "annotations": anns, "categories": [{"id": 1}, {"id": 2}]}, preds


def mots_masks(p, h=1080, w=1920, device="cuda"):
    """The detections' masks made on the device (only the update is timed, not the making)."""
    g = torch.Generator(device=device).manual_seed(p["seed"])
    n = p["n"]
    e = torch.tensor(p["ell"], dtype=torch.float32, device=device)
    pick = torch.randint(0, len(p["ell"]), (n,), generator=g, device=device)
    c = e[pick] + torch.randn(n, 4, generator=g, device=device) * torch.tensor([4.0, 4.0, 2.0, 4.0], device=device)
    yy = torch.arange(h, device=device, dtype=torch.float32)[:, None]
    xx = torch.arange(w, device=device, dtype=torch.float32)[None, :]
    masks = torch.empty(n, 1, h, w, dtype=torch.bool, device=device)
    for d in range(n):
        cx, cy, rx, ry = c[d]
        masks[d, 0] = ((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 <= 1
    return {"scores": torch.rand(n, generator=g, device=device), "labels": torch.zeros(n, dtype=torch.int64,
                                                                                       device=device),
            "masks": masks}


def run(name, ds, preds, iou_type, batch, oracle):
    dev = torch.device("cuda")
    ids = sorted(preds)
    if iou_type == "segm":
        batches = [[i] for i in ids]
    else:
        preds = {i: {k: v.to(dev) for k, v in p.items()} for i, p in preds.items()}
        batches = [ids[b:b + batch] for b in range(0, len(ids), batch)]
    for rep in range(2):                                           # the first pass warms up
        ev = ce.CocoEvaluator(ds, (iou_type,))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        t_upd = 0.0
        for bt in batches:
            if iou_type == "segm":
                upd = {i: mots_masks(preds[i]) for i in bt}
                torch.cuda.synchronize()
            else:
                upd = {i: preds[i] for i in bt}
            s = time.perf_counter()
            ev.update(upd)
            torch.cuda.synchronize()
            t_upd += time.perf_counter() - s
        ev.synchronize_between_processes()
        torch.cuda.synchronize()
        s = time.perf_counter()
        ev.accumulate()
        t_acc = time.perf_counter() - s
        t_all = time.perf_counter() - t0
    res = {"workload": name, "images": len(ids), "iou_type": iou_type, "batch": len(batches[0]),
           "update_ms_per_batch": 1e3 * t_upd / len(batches), "accumulate_ms": 1e3 * t_acc,
           "updates_total_ms": 1e3 * t_upd}
    e = ev.coco_eval[iou_type]
    res["stats"] = [round(float(x), 6) for x in ce.summarize_eval(e.eval, e.params, out=lambda s: None)]
    if iou_type == "segm":
        res["whole_ms_excluding_mask_making"] = 1e3 * (t_upd + t_acc)
    else:
        res["whole_ms"] = 1e3 * t_all
    if oracle:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import coco_eval_reference as ref
        if iou_type == "segm":
            host = {i: {k: v.cpu().numpy() for k, v in mots_masks(preds[i]).items()} for i in ids}
        else:
            host = {i: {k: v.cpu().numpy() for k, v in p.items()} for i, p in preds.items()}
        s = time.perf_counter()
        o = ref.coco_eval(ds, [host], iou_type)
        res["oracle_s"] = time.perf_counter() - s
        res["equal_to_oracle"] = bool(np.array_equal(o[0], ev.coco_eval[iou_type].eval["precision"]) and
                                      np.array_equal(o[1], ev.coco_eval[iou_type].eval["recall"]))
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="mot17,crowdhuman,coco,mots20")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--frames", type=int, default=200, help="mots20 frames")
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("coco_eval_bench needs a CUDA device")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = torch.cuda.get_device_name(0)
    print(json.dumps({"card": card}), flush=True)
    rng = np.random.default_rng(0)
    out = []
    for wl in a.workloads.split(","):
        if wl == "mot17":
            ds, p = boxes_workload(rng, 2650, 1, 30, 300)
            out.append(run(wl, ds, p, "bbox", a.batch, a.oracle))
        elif wl == "crowdhuman":
            ds, p = boxes_workload(rng, 4370, 1, 23, 100)
            out.append(run(wl, ds, p, "bbox", a.batch, a.oracle))
        elif wl == "coco":
            ds, p = boxes_workload(rng, 5000, 80, 7, 100, 480, 640)
            out.append(run(wl, ds, p, "bbox", a.batch, a.oracle))
        elif wl == "mots20":
            ds, p = mots_workload(rng, a.frames)
            out.append(run(wl, ds, p, "segm", 1, a.oracle))
        else:
            raise SystemExit(f"unknown workload {wl}")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": card, "results": out}, f, indent=1)


if __name__ == "__main__":
    main()
