"""Seeded synthetic COCO scenes for the COCO-eval tests: a ground-truth dataset dict and a list of updates
({image_id: {"scores", "labels", "boxes"[, "masks"]}} of CPU tensors), plus helpers shared by the CPU and GPU
suites."""
import numpy as np
import torch

from trackformer_b200 import mots


def _rect_mask(h, w, x0, y0, x1, y1):
    m = np.zeros((h, w), bool)
    m[max(0, y0):max(0, y1), max(0, x0):max(0, x1)] = True
    return m


def _ellipse_mask(h, w, cx, cy, rx, ry):
    yy, xx = np.mgrid[0:h, 0:w]
    return ((xx - cx) / max(rx, 1)) ** 2 + ((yy - cy) / max(ry, 1)) ** 2 <= 1.0


def scene(seed, kind="coco", segm=False, n_images=6, size=(48, 64), updates=2, dup=True):
    """kind: "coco" (several categories, a few objects each) or "mot" (one category, dense crowds with ignore
    boxes and ids from 0).  Boxes sit on a coarse grid so that equal IoUs and tied scores occur."""
    rng = np.random.default_rng(seed)
    h, w = size
    n_cat = 4 if kind == "coco" else 1
    cats = [{"id": c + 1, "name": str(c)} for c in range(n_cat)]
    if kind == "coco":
        cats.append({"id": 9, "name": "unused"})                   # a category without ground truth
    images, anns = [], []
    ann_id = 0 if kind == "mot" else 1
    for i in range(n_images):
        img_id = 10 + 3 * i
        images.append({"id": img_id, "height": h, "width": w})
        n_gt = int(rng.integers(0, 4 if kind == "coco" else 14))
        for _ in range(n_gt):
            x0, y0 = float(rng.integers(0, w - 8)), float(rng.integers(0, h - 8))
            bw, bh = float(rng.integers(2, w // 2)), float(rng.integers(2, h // 2))
            a = {"id": ann_id, "image_id": img_id, "category_id": int(rng.integers(1, n_cat + 1)),
                 "bbox": [x0, y0, bw, bh], "iscrowd": int(rng.random() < 0.1)}
            if kind == "mot":
                a["ignore"] = int(rng.random() < 0.2)
            if segm:
                m = (_ellipse_mask(h, w, x0 + bw / 2, y0 + bh / 2, bw / 2, bh / 2) if rng.random() < 0.5
                     else _rect_mask(h, w, int(x0), int(y0), int(x0 + bw), int(y0 + bh)))
                rle = mots.encode(m)
                if rng.random() < 0.5:
                    rle["counts"] = rle["counts"].decode()
                else:
                    rle["counts"] = mots.decode_counts(rle["counts"]).tolist()
                a["segmentation"] = rle
                a["area"] = float(m.sum())
            else:
                a["area"] = float(rng.choice([bw * bh, 32.0 ** 2, 96.0 ** 2, bw * bh * 0.8]))
            anns.append(a)
            ann_id += 1
    dataset = {"images": images, "annotations": anns, "categories": cats}
    ids = [im["id"] for im in images]
    ups = []
    for u in range(updates):
        pick = ids[u::updates]
        if dup and u > 0:
            pick = pick + [ids[0]]                                 # a padded duplicate, as DistributedSampler makes
        upd = {}
        for img_id in pick:
            gts = [a for a in anns if a["image_id"] == img_id]
            n = int(rng.integers(0, 130 if kind == "mot" else 25))
            boxes = np.zeros((n, 4), np.float32)
            for j in range(n):
                if gts and rng.random() < 0.7:
                    g = gts[int(rng.integers(len(gts)))]["bbox"]
                    jit = rng.integers(-2, 3, 4).astype(np.float32)
                    x0, y0 = g[0] + jit[0], g[1] + jit[1]
                    boxes[j] = (x0, y0, x0 + g[2] + jit[2], y0 + g[3] + jit[3])
                else:
                    x0, y0 = rng.integers(0, w - 4), rng.integers(0, h - 4)
                    boxes[j] = (x0, y0, x0 + rng.integers(1, w // 2), y0 + rng.integers(1, h // 2))
            scores = (rng.integers(0, 20, n) / 20.0).astype(np.float32)   # ties
            labels = rng.integers(0, n_cat, n).astype(np.int64)
            pred = {"scores": torch.from_numpy(scores), "labels": torch.from_numpy(labels),
                    "boxes": torch.from_numpy(boxes), "scores_no_object": torch.zeros(n)}
            if segm:
                masks = np.zeros((n, 1, h, w), bool)
                for j in range(n):
                    x0, y0, x1, y1 = boxes[j].astype(int)
                    r = rng.random()
                    if r < 0.1:
                        continue                                   # empty mask
                    masks[j, 0] = (_rect_mask(h, w, x0, y0, x1, y1) if r < 0.5
                                   else _ellipse_mask(h, w, (x0 + x1) / 2, (y0 + y1) / 2, (x1 - x0) / 2,
                                                      (y1 - y0) / 2))
                pred["masks"] = torch.from_numpy(masks)
            upd[img_id] = pred
        ups.append(upd)
    return dataset, ups


def as_numpy(updates):
    return [{i: {k: v.cpu().numpy() for k, v in p.items()} for i, p in u.items()} for u in updates]
