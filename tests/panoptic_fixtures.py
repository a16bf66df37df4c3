"""Synthetic panoptic scenes for the PQ tests: GT and prediction id maps made of rectangles, with crowd regions, VOID,
unlisted GT ids and category mismatches, and the `segments_info` of each side."""
import numpy as np


def categories(n_things=8, n_stuff=5):
    cats = [{"id": 1 + 2 * k, "name": f"thing{k}", "isthing": 1} for k in range(n_things)]
    cats += [{"id": 100 + k, "name": f"stuff{k}", "isthing": 0} for k in range(n_stuff)]
    return cats


def scene(seed, H=48, W=64, image_id=1, n_gt=8, n_pred=10, cats=None):
    """One image: (gt_ann, gt_map, pred_ann, pred_map)."""
    rng = np.random.default_rng(seed)
    cats = cats or categories()
    cat_ids = [c["id"] for c in cats]
    gt = np.zeros((H, W), np.int32)
    gt_ids = rng.choice(np.arange(1, 3000), n_gt, replace=False)
    gsegs = []
    for gid in gt_ids:
        y0, x0 = rng.integers(0, H - 4), rng.integers(0, W - 4)
        y1, x1 = y0 + rng.integers(3, H // 2), x0 + rng.integers(3, W // 2)
        gt[y0:y1, x0:x1] = gid
    unlisted = int(gt_ids[-1])                                  # drawn but not listed
    gcat = {}
    for gid in gt_ids[:-1]:
        a = int((gt == gid).sum())
        if a == 0:
            continue
        gcat[int(gid)] = int(rng.choice(cat_ids))
        gsegs.append({"id": int(gid), "category_id": gcat[int(gid)], "area": a,
                      "iscrowd": int(rng.random() < 0.2)})
    pred = np.zeros((H, W), np.int32)
    psegs = []
    for k in range(n_pred):
        src = [s for s in gsegs] if gsegs else []
        if src and rng.random() < 0.7:                         # a perturbed copy of a GT segment
            s = src[rng.integers(len(src))]
            ys, xs = np.nonzero(gt == s["id"])
            dy, dx = rng.integers(-3, 4, 2)
            y0, y1 = max(0, ys.min() + dy), min(H, ys.max() + 1 + dy)
            x0, x1 = max(0, xs.min() + dx), min(W, xs.max() + 1 + dx)
            cat = s["category_id"] if rng.random() < 0.85 else int(rng.choice(cat_ids))
        else:
            y0, x0 = rng.integers(0, H - 4), rng.integers(0, W - 4)
            y1, x1 = y0 + rng.integers(2, H // 3), x0 + rng.integers(2, W // 3)
            cat = int(rng.choice(cat_ids))
        pid = int(rng.integers(1, 1 << 24)) if rng.random() < 0.5 else k + 1
        if any(p["id"] == pid for p in psegs) or y1 <= y0 or x1 <= x0:
            continue
        pred[y0:y1, x0:x1] = pid
        psegs.append({"id": pid, "category_id": cat})
    present = set(np.unique(pred).tolist())
    psegs = [p for p in psegs if p["id"] in present]
    fname = f"{image_id:012d}.png"
    return ({"image_id": image_id, "file_name": fname, "segments_info": gsegs}, gt,
            {"image_id": image_id, "file_name": fname, "segments_info": psegs}, pred), unlisted


def dataset(seed, n_images, H=48, W=64, **kw):
    """(gt_json, pred_json, gt_maps, pred_maps) of n_images scenes."""
    cats = categories()
    gt_anns, pred_anns, gmaps, pmaps = [], [], {}, {}
    for i in range(n_images):
        (ga, gm, pa, pm), _ = scene(seed * 1000 + i, H, W, image_id=10 + 3 * i, cats=cats, **kw)
        gt_anns.append(ga)
        pred_anns.append(pa)
        gmaps[ga["image_id"]] = gm
        pmaps[pa["image_id"]] = pm
    return ({"categories": cats, "annotations": gt_anns, "images": []}, {"annotations": pred_anns}, gmaps, pmaps)
