"""Seeded scenes for the cross-evaluator and invariance tests (tests/test_eval_consistency_*.py), and the
transformations those tests apply to them.

Every scene is built so that the relations the tests check hold exactly, not just approximately:
  * box coordinates are integers and every box lies inside its image; a box's mask is the pixel rectangle
    [x1, x2) x [y1, y2), given as a COCO RLE written straight from its column intervals (no dense pass);
  * the objects of one frame sit in disjoint cells of a grid, so the GT masks of a frame do not overlap, and neither
    do the hypothesis masks (with disjoint masks on each side no (GT, hypothesis) assignment can tie);
  * no IoU of a candidate pair lies within 1e-6 of a threshold (COCO's 0.50 .. 0.95, MOT's and PQ's 0.5), and no two
    detection scores are equal;
  * empty frames and images, tracks with gaps, and frames with more than MAX_CLEAR_COMPONENT (64) objects occur.
numpy randomness only."""
from fractions import Fraction

import numpy as np
import torch

import mots_eval_fixtures as msf
from trackformer_b200 import mot_eval, mots, mots_eval

COCO_THRESHOLDS = [Fraction(50 + 5 * i, 100) for i in range(10)]
HALF = [Fraction(1, 2)]


def rect_iou(a, b, crowd=False):
    """Exact IoU of two [x1, y1, x2, y2] integer rectangles (a the detection); a crowd GT's union is a's area."""
    iw = max(0, min(a[2], b[2]) - max(a[0], b[0]))
    ih = max(0, min(a[3], b[3]) - max(a[1], b[1]))
    inter = iw * ih
    area_a = (a[2] - a[0]) * (a[3] - a[1])
    union = area_a if crowd else area_a + (b[2] - b[0]) * (b[3] - b[1]) - inter
    return Fraction(inter, union) if union else Fraction(0)


def clear_of(iou, thresholds):
    return all(abs(iou - t) > Fraction(1, 10 ** 6) for t in thresholds)


def rect_rle(box, h, w):
    """COCO RLE {"size", "counts" bytes} of the pixel rectangle [x1, x2) x [y1, y2) of an h x w image."""
    x1, y1, x2, y2 = (int(v) for v in box)
    iv = [(c * h + y1, c * h + y2) for c in range(x1, x2)] if x2 > x1 and y2 > y1 else []
    return msf.rle(np.asarray(iv, np.int64).reshape(-1, 2), h, w)


def rect_mask(box, h, w):
    m = np.zeros((h, w), bool)
    x1, y1, x2, y2 = (int(v) for v in box)
    m[y1:y2, x1:x2] = True
    return m


def _inner(rng, cell, lo=0.3, hi=0.9):
    """An integer rectangle inside the cell [x, y, x + cw, y + ch]."""
    x, y, cw, ch = cell
    bw = int(rng.integers(max(2, int(lo * cw)), max(3, int(hi * cw)) + 1))
    bh = int(rng.integers(max(2, int(lo * ch)), max(3, int(hi * ch)) + 1))
    x1 = x + int(rng.integers(0, cw - bw + 1))
    y1 = y + int(rng.integers(0, ch - bh + 1))
    return [x1, y1, x1 + bw, y1 + bh]


def _near(rng, gt, cell, thresholds, crowd=False, far=False, tries=64):
    """A rectangle inside the cell whose IoU with gt keeps clear of every threshold (far: often below them all)."""
    x, y, cw, ch = cell
    for _ in range(tries):
        if far:
            b = _inner(rng, cell, 0.2, 0.6)
        else:
            j = rng.integers(-3, 4, 4)
            b = [gt[0] + j[0], gt[1] + j[1], gt[2] + j[2], gt[3] + j[3]]
            b = [min(max(b[0], x), x + cw - 1), min(max(b[1], y), y + ch - 1),
                 min(max(b[2], x + 1), x + cw), min(max(b[3], y + 1), y + ch)]
            if b[2] <= b[0] or b[3] <= b[1]:
                continue
        if clear_of(rect_iou(b, gt, crowd), thresholds):
            return b
    return None


def _cells(h, w, cw, ch):
    return [(c * cw, r * ch, cw, ch) for r in range(h // ch) for c in range(w // cw)]


# ---------------------------------------------------------------- COCO

def coco_scene(seed, images=((192, 192, 16), (480, 480, 120), (240, 240, 40), (64, 96, 32), (64, 64, 32)),
               n_cat=4, many_dets=True, pad=0):
    """(dataset, update) for box and mask evaluation alike: GT annotations carry both a bbox and the RLE of its
    rectangle, area = w * h, some iscrowd = 1; the predictions carry boxes (float32 x1, y1, x2, y2) and the rectangles
    as bool masks [n, 1, h, w].  `images` are (height, width, cell): the first image has 144 cells, so one category
    gets more than 100 detections (`many_dets`); the 480 x 480 and 240 x 240 images have areas on both sides of 96^2
    and 32^2; an image without anything and one with detections but no GT come last.  Category n_cat + 3 is listed
    without GT; category n_cat + 5 is not listed.  `pad`: pixels left free round every image (so the scene can
    move).  Scores are distinct over the whole scene."""
    rng = np.random.default_rng(seed)
    cat_ids = list(range(1, n_cat + 1)) + [n_cat + 3]
    imgs, anns, preds = [], [], {}
    n_det = 0
    for i, (h, w, cs) in enumerate(images):
        img_id = 3 + 7 * i
        imgs.append({"id": img_id, "height": h, "width": w})
        boxes, labels = [], []
        empty = i == len(images) - 2
        no_gt = i == len(images) - 1
        cells = [(x + pad, y + pad, cw, ch) for x, y, cw, ch in _cells(h - 2 * pad, w - 2 * pad, cs, cs)]
        for cell in ([] if empty else cells):
            r = rng.random()
            k = 0 if (i == 0 and many_dets) else int(rng.integers(0, n_cat))
            if no_gt or r < 0.15:                                       # a detection alone (a false positive)
                b = _inner(rng, cell)
                lab = k if rng.random() < 0.8 else int(rng.choice([n_cat + 2, n_cat + 4]))   # no-GT / unlisted
                boxes.append(b)
                labels.append(lab)
                continue
            gt = _inner(rng, cell, 0.5, 0.85)
            crowd = int(rng.random() < 0.1)
            anns.append({"id": len(anns) + 1, "image_id": img_id, "category_id": k + 1,
                         "bbox": [float(gt[0]), float(gt[1]), float(gt[2] - gt[0]), float(gt[3] - gt[1])],
                         "area": float((gt[2] - gt[0]) * (gt[3] - gt[1])), "iscrowd": crowd,
                         "segmentation": _coco_rle(gt, h, w, len(anns))})
            if r < 0.25:
                continue                                                # missed
            if crowd:                                                   # two disjoint detections inside the crowd
                xm = (gt[0] + gt[2]) // 2
                for b in ([gt[0], gt[1], xm, gt[3]], [xm, gt[1], gt[2], gt[3]]):
                    if b[2] > b[0]:
                        boxes.append(b)
                        labels.append(k)
                continue
            b = _near(rng, gt, cell, COCO_THRESHOLDS, far=r > 0.85)
            if b is not None:
                boxes.append(b)
                labels.append(k if rng.random() < 0.9 else (k + 1) % n_cat)
        n = len(boxes)
        preds[img_id] = (np.asarray(boxes, np.int64).reshape(-1, 4), np.asarray(labels, np.int64), (h, w))
        n_det += n
    order = rng.permutation(n_det)
    values = ((order + 1) / (n_det + 1)).astype(np.float32)
    assert len(np.unique(values)) == n_det
    update, at = {}, 0
    for img_id, (boxes, labels, (h, w)) in preds.items():
        n = len(boxes)
        masks = np.zeros((n, 1, h, w), bool)
        for j, b in enumerate(boxes):
            masks[j, 0] = rect_mask(b, h, w)
        update[img_id] = {"scores": torch.from_numpy(values[at:at + n].copy()),
                          "labels": torch.from_numpy(labels.copy()),
                          "boxes": torch.from_numpy(boxes.astype(np.float32)),
                          "masks": torch.from_numpy(masks)}
        at += n
    dataset = {"images": imgs, "annotations": anns, "categories": [{"id": c, "name": str(c)} for c in cat_ids]}
    return dataset, update


def _coco_rle(box, h, w, n):
    """The rectangle's RLE in both forms coco_eval reads: a counts string, or (every other annotation) a list."""
    r = rect_rle(box, h, w)
    counts = r["counts"].decode()
    if n % 2:
        return {"size": [h, w], "counts": mots.decode_counts(counts).tolist()}
    return {"size": [h, w], "counts": counts}


def coco_relabel(dataset, update, rng, cats=True, anns=True, images=True):
    """Random injective maps of category, annotation and image ids (annotation ids avoid 0: pycocotools does not
    count a match to annotation id 0 as a true positive, so 0 is not a free label).  Returns the new scene and the
    new category index of each old one."""
    old_cats = sorted(c["id"] for c in dataset["categories"])
    new_c = rng.choice(np.arange(1, 1000), len(old_cats), replace=False) if cats else np.asarray(old_cats)
    cmap = {o: int(n) for o, n in zip(old_cats, new_c)}
    amap = dict(zip([a["id"] for a in dataset["annotations"]],
                    (rng.choice(np.arange(1, 10 ** 6), len(dataset["annotations"]), replace=False) if anns
                     else [a["id"] for a in dataset["annotations"]])))
    img_ids = [im["id"] for im in dataset["images"]]
    imap = dict(zip(img_ids, (rng.choice(np.arange(10 ** 6), len(img_ids), replace=False) if images else img_ids)))
    ds = {"images": [dict(im, id=int(imap[im["id"]])) for im in dataset["images"]],
          "annotations": [dict(a, id=int(amap[a["id"]]), image_id=int(imap[a["image_id"]]),
                               category_id=cmap[a["category_id"]]) for a in dataset["annotations"]],
          "categories": [dict(c, id=cmap[c["id"]]) for c in dataset["categories"]]}

    def label(lb):                               # labels are category id - 1; unlisted labels stay unlisted
        return torch.tensor([cmap[int(v) + 1] - 1 if int(v) + 1 in cmap else 5000 + int(v) for v in lb],
                            dtype=torch.int64)

    up = {int(imap[i]): dict(p, labels=label(p["labels"])) for i, p in update.items()}
    new_sorted = sorted(cmap.values())
    k_of = np.asarray([new_sorted.index(cmap[c]) for c in old_cats])
    return ds, up, k_of


def coco_permute(update, rng):
    """The detections of every image in a random order."""
    out = {}
    for i, p in update.items():
        perm = torch.from_numpy(rng.permutation(len(p["scores"])))
        out[i] = {k: v[perm] for k, v in p.items()}
    return out


def coco_translate(dataset, update, dx, dy):
    """Every box and mask moved by (dx, dy) pixels; the caller keeps everything inside the images."""
    hw = {im["id"]: (im["height"], im["width"]) for im in dataset["images"]}
    anns = []
    for a in dataset["annotations"]:
        x, y, bw, bh = a["bbox"]
        box = [int(x) + dx, int(y) + dy, int(x + bw) + dx, int(y + bh) + dy]
        h, w = hw[a["image_id"]]
        assert 0 <= box[0] and 0 <= box[1] and box[2] <= w and box[3] <= h
        anns.append(dict(a, bbox=[float(box[0]), float(box[1]), bw, bh],
                         segmentation=_coco_rle(box, h, w, a["id"])))
    up = {}
    for i, p in update.items():
        h, w = hw[i]
        boxes = p["boxes"] + torch.tensor([dx, dy, dx, dy], dtype=torch.float32)
        assert (boxes[:, 0] >= 0).all() and (boxes[:, 1] >= 0).all() and (boxes[:, 2] <= w).all() \
            and (boxes[:, 3] <= h).all()
        masks = torch.roll(p["masks"], shifts=(dy, dx), dims=(2, 3))
        up[i] = dict(p, boxes=boxes, masks=masks)
    return dict(dataset, annotations=anns), up


def coco_margin(dataset, update):
    """(left, top, right, bottom): how far the scene can move in each direction and stay inside its images."""
    hw = {im["id"]: (im["height"], im["width"]) for im in dataset["images"]}
    m = [10 ** 9] * 4
    boxes = [(a["image_id"], [a["bbox"][0], a["bbox"][1], a["bbox"][0] + a["bbox"][2], a["bbox"][1] + a["bbox"][3]])
             for a in dataset["annotations"]]
    boxes += [(i, b.tolist()) for i, p in update.items() for b in p["boxes"]]
    for i, b in boxes:
        h, w = hw[i]
        m = [min(m[0], b[0]), min(m[1], b[1]), min(m[2], w - b[2]), min(m[3], h - b[3])]
    return [int(v) for v in m]


# ---------------------------------------------------------------- MOT and MOTS

def track_scene(seed, n_frames=12, size=(96, 160), cell=(16, 16), p_obj=0.6, p_miss=0.1, p_far=0.1, p_fp=0.1,
                p_switch=0.05, p_gap=0.1, empty_frames=(3,), ignore=False):
    """One sequence on a grid of cells: each cell holds one object slot whose GT id changes now and then; the
    object's rectangle jitters inside the cell; its hypothesis is a jittered copy (p_far: mostly a non-candidate),
    missing at times (track gaps), and its track id is swapped with another slot's now and then.  Free cells get false
    positives.  `ignore`: some free cells get an ignore region (class 10) next to a hypothesis that lies in it by less
    than, exactly, or more than half, and some objects get an ignore region beside them that their non-candidate
    hypothesis reaches into.

    Returns dict(boxes=(results, frames) for mot_eval, masks=(results, gt, n_frames) for mots_eval, size, ignore
    rectangles {frame: [box]}); the two share GT ids, track ids and the tracks' order."""
    h, w = size
    rng = np.random.default_rng(seed)
    cells = _cells(h, w, *cell)
    n = len(cells)
    slot_gt = np.arange(n) + 1
    next_gt = n + 1
    slot_track = rng.permutation(n) + 100
    next_track = 100 + n
    alive = rng.random(n) < p_obj
    gt_rows = {}                      # gid -> {f: box}
    hyp_rows = {}                     # tid -> {f: box}
    ign_rows = {}                     # f -> [box]
    frames = []
    for f in range(n_frames):
        flip = rng.random(n) < 0.1
        alive ^= flip
        for k in np.nonzero(flip & alive)[0]:                     # an object (re)enters: a new GT id
            slot_gt[k], next_gt = next_gt, next_gt + 1
        for k in np.nonzero(rng.random(n) < p_switch)[0]:
            j = rng.integers(n)
            slot_track[k], slot_track[j] = slot_track[j], slot_track[k]
        gt = {}
        if f in empty_frames:
            frames.append({"gt": gt})
            continue
        for k in rng.permutation(n):
            c = cells[k]
            if not alive[k]:
                r = rng.random()
                if ignore and r < 0.3:                            # an ignore region and a hypothesis partly in it
                    x, y, cw, ch = c
                    iw = int(rng.integers(2, cw // 2 + 1))
                    ign = [x, y + 2, x + iw, y + ch - 2]
                    hw_ = 2 * int(rng.integers(1, iw + 1))          # even width: some hypotheses exactly half in
                    inside = int(rng.choice([hw_ // 2 - 1, hw_ // 2, hw_ // 2, hw_ // 2 + 1]))
                    inside = min(max(inside, 0), iw, hw_)
                    hx = x + iw - inside
                    if hx + hw_ > x + cw:
                        continue
                    ign_rows.setdefault(f, []).append(ign)
                    hyp_rows.setdefault(int(next_track), {})[f] = [hx, y + 3, hx + hw_, y + ch - 3]
                    next_track += 1
                elif r < 0.3 + p_fp:
                    hyp_rows.setdefault(int(next_track), {})[f] = _inner(rng, c)
                    next_track += 1
                continue
            x, y, cw, ch = c
            if ignore and rng.random() < 0.3:                     # the object on the left, an ignore strip right
                sub = (x, y, cw - 5, ch)
                g = _inner(rng, sub, 0.5, 0.9)
                ign_rows.setdefault(f, []).append([x + cw - 4, y, x + cw, y + ch])
                gt[int(slot_gt[k])] = g
                gt_rows.setdefault(int(slot_gt[k]), {})[f] = g
                if rng.random() < 0.5:                            # a non-candidate reaching into the strip
                    hb = [max(g[2] - 1, x + cw - 6), y + 1, x + cw, y + ch - 1]
                    if clear_of(rect_iou(hb, g), HALF) and rect_iou(hb, g) < Fraction(1, 2):
                        hyp_rows.setdefault(int(slot_track[k]), {})[f] = hb
                        continue
                b = _near(rng, g, sub, HALF)
                if b is not None:
                    hyp_rows.setdefault(int(slot_track[k]), {})[f] = b
                continue
            g = _inner(rng, c, 0.5, 0.9)
            gt[int(slot_gt[k])] = g
            gt_rows.setdefault(int(slot_gt[k]), {})[f] = g
            if rng.random() < p_miss or rng.random() < p_gap:
                continue
            b = _near(rng, g, c, HALF, far=rng.random() < p_far)
            if b is not None:
                hyp_rows.setdefault(int(slot_track[k]), {})[f] = b
        frames.append({"gt": gt})
    order = list(hyp_rows)
    rng.shuffle(order)
    hyp_rows = {t: hyp_rows[t] for t in order}                    # tracks in no particular id order
    return build_track_scene(frames, hyp_rows, ign_rows, size)


def build_track_scene(frames, hyp_rows, ign_rows, size):
    """The MOT and MOTS inputs of one sequence given as GT frames [{"gt": {gid: box}}], hypotheses {tid: {f: box}}
    and ignore regions {f: [box]} (boxes are integer [x1, y1, x2, y2])."""
    h, w = size
    f32 = lambda b: np.asarray(b, np.float32)
    mot_results = {t: {f: {"bbox": f32(b)} for f, b in tr.items()} for t, tr in hyp_rows.items()}
    mot_frames = [{"gt": {g: f32(b) for g, b in fr["gt"].items()}} for fr in frames]
    gt = {}
    for f, fr in enumerate(frames):
        for g, b in fr["gt"].items():
            gt.setdefault(g, {})[f] = {"mask": rect_rle(b, h, w), "class_id": 2}
    for f, boxes in ign_rows.items():
        for j, b in enumerate(boxes):
            gt.setdefault(10 ** 6 + j, {})[f] = {"mask": rect_rle(b, h, w), "class_id": 10}
    mots_results = {t: {f: {"mask": rect_rle(b, h, w)} for f, b in tr.items()} for t, tr in hyp_rows.items()}
    return dict(boxes=(mot_results, mot_frames), masks=(mots_results, gt, len(frames)), size=size,
                frames=frames, hyps=hyp_rows, ignore=ign_rows)


def track_scenes(seed):
    """{name: scene}: several sequences of different sizes and lengths, one with an empty first frame, one crowded
    (99 objects in a frame), one with no hypotheses at all and one with no GT."""
    s = {"small": track_scene(seed, n_frames=9, empty_frames=(0, 4)),
         "long": track_scene(seed + 1, n_frames=30, size=(64, 128), p_switch=0.1),
         "crowded": track_scene(seed + 2, n_frames=6, size=(176, 144), p_obj=0.95, empty_frames=()),
         "wide": track_scene(seed + 3, n_frames=8, size=(48, 240), cell=(24, 16))}
    base = track_scene(seed + 4, n_frames=5, size=(32, 64))
    s["no_hyps"] = build_track_scene(base["frames"], {}, {}, base["size"])
    s["no_gt"] = build_track_scene([{"gt": {}} for _ in base["frames"]], base["hyps"], {}, base["size"])
    return s


def max_objects_per_frame(scene):
    return max(len(fr["gt"]) for fr in scene["frames"])


def relabel_track_scene(scene, rng):
    """Random injective maps of GT ids and track ids (the dicts keep their order)."""
    gids = sorted({g for fr in scene["frames"] for g in fr["gt"]})
    gmap = dict(zip(gids, (int(v) for v in rng.choice(np.arange(1, 10 ** 6), len(gids), replace=False))))
    tids = list(scene["hyps"])
    tmap = dict(zip(tids, (int(v) for v in rng.choice(np.arange(10 ** 6), len(tids), replace=False))))
    frames = [{"gt": {gmap[g]: b for g, b in fr["gt"].items()}} for fr in scene["frames"]]
    hyps = {tmap[t]: tr for t, tr in scene["hyps"].items()}
    return build_track_scene(frames, hyps, scene["ignore"], scene["size"])


def permute_tracks(scene, rng):
    tids = list(scene["hyps"])
    hyps = {tids[i]: scene["hyps"][tids[i]] for i in rng.permutation(len(tids))}
    return build_track_scene(scene["frames"], hyps, scene["ignore"], scene["size"])


def translate_track_scene(scene, dx, dy):
    mv = lambda b: [b[0] + dx, b[1] + dy, b[2] + dx, b[3] + dy]
    frames = [{"gt": {g: mv(b) for g, b in fr["gt"].items()}} for fr in scene["frames"]]
    hyps = {t: {f: mv(b) for f, b in tr.items()} for t, tr in scene["hyps"].items()}
    ign = {f: [mv(b) for b in bs] for f, bs in scene["ignore"].items()}
    return build_track_scene(frames, hyps, ign, scene["size"])


def track_margin(scene):
    h, w = scene["size"]
    boxes = [b for fr in scene["frames"] for b in fr["gt"].values()]
    boxes += [b for tr in scene["hyps"].values() for b in tr.values()]
    boxes += [b for bs in scene["ignore"].values() for b in bs]
    return [min(b[0] for b in boxes), min(b[1] for b in boxes), min(w - b[2] for b in boxes),
            min(h - b[3] for b in boxes)]


def _dense_frames(scene):
    """Per frame with hypotheses: (GT label map (index + 1 into the frame's GT boxes, 0 for none), ignore union)."""
    h, w = scene["size"]
    frames = {f for tr in scene["hyps"].values() for f in tr}
    out = {}
    for f in frames:
        lab = np.zeros((h, w), np.int32)
        for k, b in enumerate(scene["frames"][f]["gt"].values()):
            lab[b[1]:b[3], b[0]:b[2]] = k + 1
        ign = np.zeros((h, w), bool)
        for b in scene["ignore"].get(f, []):
            ign[b[1]:b[3], b[0]:b[2]] = True
        out[f] = (lab, ign)
    return out


def _ignore_counts(scene):
    """{(frame, track id): (has a candidate, pixels, pixels inside the ignore union)} from dense numpy masks: the
    hypothesis' pixels are its rectangle's; a GT is a candidate iff inter > 0 and 2 inter >= union."""
    dense = _dense_frames(scene)
    out = {}
    for t, tr in scene["hyps"].items():
        for f, b in tr.items():
            lab, ign = dense[f]
            gts = list(scene["frames"][f]["gt"].values())
            px = (b[2] - b[0]) * (b[3] - b[1])
            ids, inter = np.unique(lab[b[1]:b[3], b[0]:b[2]], return_counts=True)
            cand = False
            for k, i in zip(ids, inter):
                if k:
                    g = gts[k - 1]
                    union = px + (g[2] - g[0]) * (g[3] - g[1]) - int(i)
                    cand |= 2 * int(i) >= union
            out[(f, t)] = (cand, px, int(ign[b[1]:b[3], b[0]:b[2]].sum()))
    return out


def removed_hypotheses(scene):
    """{(frame, track id)} of the hypotheses the MOTS ignore rule removes: no candidate, and more than half of the
    pixels inside the union of the frame's ignore regions."""
    return {k for k, (cand, px, inside) in _ignore_counts(scene).items() if not cand and 2 * inside > px}


def exactly_half_inside(scene):
    """{(frame, track id)} of hypotheses with no candidate that lie exactly half inside the ignore union."""
    return {k for k, (cand, px, inside) in _ignore_counts(scene).items() if not cand and 2 * inside == px}


def without(scene, drop, ignore=False):
    """The scene without the (frame, track id) hypotheses in `drop` and (ignore=False) without ignore regions."""
    hyps = {}
    for t, tr in scene["hyps"].items():
        kept = {f: b for f, b in tr.items() if (f, t) not in drop}
        if kept:
            hyps[t] = kept
    return build_track_scene(scene["frames"], hyps, scene["ignore"] if ignore else {}, scene["size"])


def mot_accums(scenes):
    return [mot_eval.get_mot_accum(*s["boxes"]) for s in scenes.values()]


def mots_accums(scenes):
    return [mots_eval.get_mots_accum(*s["masks"]) for s in scenes.values()]


# ---------------------------------------------------------------- panoptic

def pq_categories():
    return ([{"id": 1 + 2 * k, "name": f"thing{k}", "isthing": 1} for k in range(5)]
            + [{"id": 60 + k, "name": f"stuff{k}", "isthing": 0} for k in range(3)])


def pq_scene(seed, n_images=4, size=(64, 96), cell=16, margin=8):
    """(gt_json, pred_json, gt_maps, pred_maps): id maps of rectangles in disjoint cells, a `margin`-pixel VOID frame
    round each image (so the content can move), crowd GT (at most one per image and category: panopticapi keeps the
    last crowd of a category in JSON order, so with two the order of segments_info would matter by design), a GT id
    in the map but not listed, category mismatches, predictions over VOID and over crowds, an image without
    predictions and one without GT.  Every (GT, prediction) IoU of equal categories keeps clear of 0.5."""
    rng = np.random.default_rng(seed)
    cats = pq_categories()
    cat_ids = [c["id"] for c in cats]
    h, w = size
    gt_anns, pred_anns, gmaps, pmaps = [], [], {}, {}
    for i in range(n_images):
        image_id = 5 + 4 * i
        for _ in range(100):
            gm, pm = np.zeros((h, w), np.int32), np.zeros((h, w), np.int32)
            gsegs, psegs, crowd_cats = [], [], set()
            gids = rng.choice(np.arange(1, 1 << 20), 64, replace=False)
            pids = rng.choice(np.arange(1, 1 << 24), 64, replace=False)
            ok = True
            for k, (x, y, cw, ch) in enumerate(_cells(h - 2 * margin, w - 2 * margin, cell, cell)):
                c = (x + margin, y + margin, cw, ch)
                r = rng.random()
                cat = int(rng.choice(cat_ids))
                if i == n_images - 1 or r < 0.15:                  # a prediction alone
                    if i != n_images - 2:
                        b = _inner(rng, c)
                        pm[b[1]:b[3], b[0]:b[2]] = pids[k]
                        psegs.append({"id": int(pids[k]), "category_id": cat})
                    continue
                g = _inner(rng, c, 0.5, 0.9)
                gm[g[1]:g[3], g[0]:g[2]] = gids[k]
                crowd = int(cat not in crowd_cats and rng.random() < 0.15)
                if crowd:
                    crowd_cats.add(cat)
                if r < 0.2:
                    continue                                        # drawn, not listed
                gsegs.append({"id": int(gids[k]), "category_id": cat, "area": (g[2] - g[0]) * (g[3] - g[1]),
                              "iscrowd": crowd})
                if r < 0.3 or i == n_images - 2:
                    continue                                        # missed
                b = _near(rng, g, c, HALF, far=r > 0.85) if not crowd else _inner(rng, c, 0.2, 0.5)
                if b is None:
                    ok = False
                    break
                pm[b[1]:b[3], b[0]:b[2]] = pids[k]
                psegs.append({"id": int(pids[k]), "category_id": cat if rng.random() < 0.9
                              else int(rng.choice(cat_ids))})
            if ok and _pq_clear(gm, pm, gsegs, psegs):
                break
        fname = f"{image_id:012d}.png"
        gt_anns.append({"image_id": image_id, "file_name": fname, "segments_info": gsegs})
        pred_anns.append({"image_id": image_id, "file_name": fname, "segments_info": psegs})
        gmaps[image_id], pmaps[image_id] = gm, pm
    return ({"categories": cats, "annotations": gt_anns, "images": []}, {"annotations": pred_anns}, gmaps, pmaps)


def _pq_clear(gm, pm, gsegs, psegs):
    """panopticapi's IoU (union less the prediction's VOID pixels) of every pair keeps clear of 0.5."""
    for g in gsegs:
        if g["iscrowd"]:
            continue
        gmask = gm == g["id"]
        for p in psegs:
            pmask = pm == p["id"]
            inter = int((gmask & pmask).sum())
            if inter == 0:
                continue
            union = int(pmask.sum()) + g["area"] - inter - int((pmask & (gm == 0)).sum())
            if not clear_of(Fraction(inter, union), HALF):
                return False
    return True


def pq_relabel(data, rng, gt_ids=True, pred_ids=True, cats=True):
    """Random injective maps of category ids, prediction segment ids and GT segment ids.  The GT map is increasing:
    panopticapi adds an image's IoUs in ascending GT id, so another order of GT ids could change the last bit of an
    fp64 sum; the counts do not depend on it."""
    gt_json, pred_json, gmaps, pmaps = data
    cmap = {c["id"]: int(n) for c, n in zip(gt_json["categories"],
                                          rng.choice(np.arange(1, 5000), len(gt_json["categories"]), replace=False))}
    if not cats:
        cmap = {c: c for c in cmap}
    g_new, p_new = {}, {}
    ga, pa = [], []
    for g_ann, p_ann in zip(gt_json["annotations"], pred_json["annotations"]):
        iid = g_ann["image_id"]
        gu = [int(v) for v in np.unique(gmaps[iid]) if v]
        pu = [int(v) for v in np.unique(pmaps[iid]) if v]
        gnew = np.sort(rng.choice(np.arange(1, 1 << 24), len(gu), replace=False)) if gt_ids else np.asarray(gu)
        pnew = rng.choice(np.arange(1, 1 << 24), len(pu), replace=False) if pred_ids else np.asarray(pu)
        gm_, pm_ = dict(zip(gu, (int(v) for v in gnew))), dict(zip(pu, (int(v) for v in pnew)))
        g_new[iid] = _remap(gmaps[iid], gm_)
        p_new[iid] = _remap(pmaps[iid], pm_)
        ga.append(dict(g_ann, segments_info=[dict(s, id=gm_[s["id"]], category_id=cmap[s["category_id"]])
                                             for s in g_ann["segments_info"]]))
        pa.append(dict(p_ann, segments_info=[dict(s, id=pm_[s["id"]], category_id=cmap[s["category_id"]])
                                             for s in p_ann["segments_info"]]))
    cats_new = [dict(c, id=cmap[c["id"]]) for c in gt_json["categories"]]
    return (dict(gt_json, categories=cats_new, annotations=ga), {"annotations": pa}, g_new, p_new), cmap


def _remap(m, mp):
    out = np.zeros_like(m)
    for o, n in mp.items():
        out[m == o] = n
    return out


def pq_permute(data, rng):
    """segments_info of both sides in a random order."""
    gt_json, pred_json, gmaps, pmaps = data
    shuf = lambda segs: [segs[i] for i in rng.permutation(len(segs))]
    gt_anns = [dict(a, segments_info=shuf(a["segments_info"])) for a in gt_json["annotations"]]
    return (dict(gt_json, annotations=gt_anns),
            {"annotations": [dict(a, segments_info=shuf(a["segments_info"])) for a in pred_json["annotations"]]},
            gmaps, pmaps)


def pq_translate(data, dy, dx, margin=8):
    """Both maps of every image moved by (dx, dy) pixels, inside the VOID margin."""
    gt_json, pred_json, gmaps, pmaps = data
    for m in list(gmaps.values()) + list(pmaps.values()):
        assert not m[:margin].any() and not m[-margin:].any() and not m[:, :margin].any() and not m[:, -margin:].any()
    mv = lambda m: np.roll(m, (dy, dx), axis=(0, 1))
    return gt_json, pred_json, {i: mv(m) for i, m in gmaps.items()}, {i: mv(m) for i, m in pmaps.items()}
