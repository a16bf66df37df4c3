"""Plain numpy / Python restatement of pycocotools 2.0's COCOeval (`evaluate`, `evaluateImg`, `accumulate`,
`summarize`) as the reference's CocoEvaluator drives it (datasets/coco_eval.py: per-update `evaluate`, then `merge`
of every update's per-image results, keeping the first occurrence of an image id).  The oracle of the COCO-eval tests;
pinned by the hand-worked scenes of tests/test_coco_eval_cpu.py.

Predictions are what `update` takes: {image_id: {"scores", "labels", "boxes" float32 x0, y0, x1, y1 [, "masks"
bool [N, 1, H, W]]}} of numpy arrays.  Ground-truth masks are RLE dicts, decoded with numpy here."""
import numpy as np

from trackformer_b200 import mots

IOU_THRS = np.linspace(.5, 0.95, 10)
REC_THRS = np.linspace(.0, 1.00, 101)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]


def _gt_mask(ann, h, w):
    seg = ann["segmentation"]
    c = seg["counts"]
    if isinstance(c, list):
        cnts = np.asarray(c, np.int64)
        return np.repeat(np.arange(len(cnts)) % 2 == 1, cnts).reshape(w, h).T
    return mots.decode(seg)


def box_iou(d, g, crowd):
    """maskApi.c bbIou on [x, y, w, h] doubles."""
    w = min(d[2] + d[0], g[2] + g[0]) - max(d[0], g[0])
    if w <= 0:
        return 0.0
    h = min(d[3] + d[1], g[3] + g[1]) - max(d[1], g[1])
    if h <= 0:
        return 0.0
    i = w * h
    u = d[2] * d[3] if crowd else d[2] * d[3] + g[2] * g[3] - i
    return i / u


def mask_iou(dm, gm, crowd):
    i = int(np.count_nonzero(dm & gm))
    if i == 0:
        return 0.0
    u = int(np.count_nonzero(dm)) if crowd else int(np.count_nonzero(dm | gm))
    return i / u


def evaluate_update(dataset, predictions, iou_type):
    """One update: {image_id: {cat_id: evalImg dict or None per area range}} over the update's images."""
    cats = sorted(c["id"] for c in dataset["categories"])
    imgs = {im["id"]: im for im in dataset["images"]}
    out = {}
    for img_id in sorted(predictions):
        im = imgs[img_id]
        h, w = im.get("height", 0), im.get("width", 0)
        pred = predictions[img_id]
        dts = []
        for n in range(len(pred["scores"])):
            cat = int(pred["labels"][n]) + 1
            d = {"score": float(np.float32(pred["scores"][n])), "category_id": cat}
            if iou_type == "bbox":
                b = np.asarray(pred["boxes"][n], np.float32)
                d["bbox"] = [float(b[0]), float(b[1]), float(np.float32(b[2] - b[0])), float(np.float32(b[3] - b[1]))]
                d["area"] = d["bbox"][2] * d["bbox"][3]
            else:
                d["mask"] = np.asarray(pred["masks"][n, 0]) > 0.5
                d["area"] = int(np.count_nonzero(d["mask"]))
            dts.append(d)
        gts = [a for a in dataset["annotations"] if a["image_id"] == img_id]
        per_cat = {}
        for cat in cats:
            gt = [g for g in gts if g["category_id"] == cat]
            dt = [d for d in dts if d["category_id"] == cat]
            if not gt and not dt:
                per_cat[cat] = None
                continue
            order = np.argsort([-d["score"] for d in dt], kind="mergesort")
            dt = [dt[i] for i in order][:MAX_DETS[-1]]
            crowd = [int(g.get("iscrowd", 0)) for g in gt]
            ious = np.zeros((len(dt), len(gt)))
            for di, d in enumerate(dt):
                for gi, g in enumerate(gt):
                    if iou_type == "bbox":
                        ious[di, gi] = box_iou(d["bbox"], [float(v) for v in g["bbox"]], crowd[gi])
                    else:
                        ious[di, gi] = mask_iou(d["mask"], _gt_mask(g, h, w), crowd[gi])
            per_cat[cat] = [evaluate_img(dt, gt, ious, crowd, rng) for rng in AREA_RNG]
        out[img_id] = per_cat
    return out


def evaluate_img(dt, gt, ious, crowd, rng):
    ignore = [1 if (c or g["area"] < rng[0] or g["area"] > rng[1]) else 0 for g, c in zip(gt, crowd)]
    gtind = np.argsort(ignore, kind="mergesort")
    gt_ig = np.asarray([ignore[i] for i in gtind])
    crowd_s = [crowd[i] for i in gtind]
    ids = [gt[i]["id"] for i in gtind]
    T = len(IOU_THRS)
    gtm = np.zeros((T, len(gt)))
    dtm = np.zeros((T, len(dt)))
    dt_ig = np.zeros((T, len(dt)))
    for tind, t in enumerate(IOU_THRS):
        for dind in range(len(dt)):
            iou = min([t, 1 - 1e-10])
            m = -1
            for g in range(len(gtind)):
                if gtm[tind, g] > 0 and not crowd_s[g]:
                    continue
                if m > -1 and gt_ig[m] == 0 and gt_ig[g] == 1:
                    break
                if ious[dind, gtind[g]] < iou:
                    continue
                iou = ious[dind, gtind[g]]
                m = g
            if m == -1:
                continue
            dt_ig[tind, dind] = gt_ig[m]
            dtm[tind, dind] = ids[m]
            gtm[tind, m] = dind + 1
    a = np.array([d["area"] < rng[0] or d["area"] > rng[1] for d in dt]).reshape((1, len(dt)))
    dt_ig = np.logical_or(dt_ig, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
    return {"dtMatches": dtm, "dtScores": [d["score"] for d in dt], "gtIgnore": gt_ig, "dtIgnore": dt_ig}


def merge(per_update):
    """The reference's merge: the first occurrence of every image id over the updates (already in rank order)."""
    kept = {}
    for upd in per_update:
        for img_id, v in upd.items():
            kept.setdefault(img_id, v)
    return dict(sorted(kept.items()))


def accumulate(dataset, evals):
    cats = sorted(c["id"] for c in dataset["categories"])
    T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(cats), len(AREA_RNG), len(MAX_DETS)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    scores = -np.ones((T, R, K, A, M))
    for k, cat in enumerate(cats):
        for a in range(A):
            E = [ev[cat][a] for ev in evals.values() if ev[cat] is not None]
            if not E:
                continue
            for m, max_det in enumerate(MAX_DETS):
                dt_scores = np.concatenate([e["dtScores"][0:max_det] for e in E])
                inds = np.argsort(-dt_scores, kind="mergesort")
                sorted_scores = dt_scores[inds]
                dtm = np.concatenate([e["dtMatches"][:, 0:max_det] for e in E], axis=1)[:, inds]
                dt_ig = np.concatenate([e["dtIgnore"][:, 0:max_det] for e in E], axis=1)[:, inds]
                gt_ig = np.concatenate([e["gtIgnore"] for e in E])
                npig = np.count_nonzero(gt_ig == 0)
                if npig == 0:
                    continue
                tps = np.logical_and(dtm, np.logical_not(dt_ig))
                fps = np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig))
                tp_sum = np.cumsum(tps, axis=1).astype(np.float64)
                fp_sum = np.cumsum(fps, axis=1).astype(np.float64)
                for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                    nd = len(tp)
                    rc = tp / npig
                    pr = (tp / (fp + tp + np.spacing(1))).tolist()
                    q = [0.0] * R
                    ss = [0.0] * R
                    recall[t, k, a, m] = rc[-1] if nd else 0
                    for i in range(nd - 1, 0, -1):
                        if pr[i] > pr[i - 1]:
                            pr[i - 1] = pr[i]
                    pinds = np.searchsorted(rc, REC_THRS, side="left")
                    try:
                        for ri, pi in enumerate(pinds):
                            q[ri] = pr[pi]
                            ss[ri] = sorted_scores[pi]
                    except IndexError:
                        pass
                    precision[t, :, k, a, m] = np.array(q)
                    scores[t, :, k, a, m] = np.array(ss)
    return precision, recall, scores


def summarize(precision, recall):
    def one(ap=1, iou_thr=None, area="all", max_dets=100):
        aind = [i for i, lbl in enumerate(AREA_LBL) if lbl == area]
        mind = [i for i, md in enumerate(MAX_DETS) if md == max_dets]
        s = precision if ap == 1 else recall
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])

    return np.array([one(1), one(1, .5), one(1, .75), one(1, area="small"), one(1, area="medium"),
                     one(1, area="large"), one(0, max_dets=1), one(0, max_dets=10), one(0), one(0, area="small"),
                     one(0, area="medium"), one(0, area="large")])


def coco_eval(dataset, updates, iou_type):
    """(precision, recall, scores, stats) of a sequence of updates (rank order, then update order)."""
    evals = merge([evaluate_update(dataset, u, iou_type) for u in updates])
    precision, recall, scores = accumulate(dataset, evals)
    return precision, recall, scores, summarize(precision, recall)
