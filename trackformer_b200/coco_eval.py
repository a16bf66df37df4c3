"""COCO box and mask AP on the GPU, in place of the reference's pycocotools-based `CocoEvaluator`
(src/trackformer/datasets/coco_eval.py), which `engine.evaluate` uses to score the detector every evaluation epoch.

`CocoEvaluator(coco_gt, iou_types)` has the reference's methods.  The ground truth is packed once at construction and
uploaded once.  `update(predictions)` enqueues, per IoU type, the IoU and matching work of pycocotools' `evaluate` /
`evaluateImg` for its images (csrc/coco_eval.cu) and keeps a compact per-detection record on the device: its sort
key, its score rank within (image, category) and a 2-bit true-positive / false-positive / ignored state per area
range and IoU threshold.  It does not synchronise with the host.  `synchronize_between_processes()` keeps the first
record of every image id over the ranks, as the reference's `merge` does.  `accumulate()` makes one C-entry call over
the kept images and one read-back of pycocotools' `precision` / `recall` / `scores` arrays.  `summarize()` prints and
sets `stats` on the host.

The numbers are those of pycocotools 2.0's `COCOeval` with its default parameters, as the reference calls it,
including its quirks: an annotation's own `ignore` key is replaced by `iscrowd`, and a detection matched to an
annotation with id 0 is not a true positive.  Ground-truth masks may be RLEs (compressed or not) or polygon and
box lists, which `COCO.annToRLE` rasterises: `CocoEvaluator` packs every polygon of the segm ground truth once and
rasterises them in one call on its device (trackformer_b200.coco_masks, csrc/coco_poly.cu), bit for bit as
pycocotools' `frPyObjects` + `merge`; an annotation's `area` still comes from the JSON.  `GroundTruth(dataset, True)`
without a device rejects polygons.  Keypoints are not supported, and pycocotools' per-image `evalImgs` dicts are not
built.  CUDA only: there is no host fallback.
"""
from __future__ import annotations

import copy
import ctypes
import datetime
import json
import os

import numpy as np
import torch

from . import coco_masks, mots

__all__ = ["CocoEvaluator", "Params", "GroundTruth", "kept_images", "MAX_DETS_PER_IMAGE", "MAX_GT_PER_IMAGE_CATEGORY"]

MAX_DETS_PER_IMAGE = 4096           # TFB200_COCO_MAX_DETS (include/tfb200_fused.h)
MAX_GT_PER_IMAGE_CATEGORY = 4096    # TFB200_COCO_MAX_GT
IOU_TYPES = ("bbox", "segm")
_IMG_FIELDS = 10


class Params:
    """pycocotools' default detection parameters (`Params.setDetParams`)."""

    def __init__(self, iouType="bbox", catIds=(), imgIds=()):
        self.iouType = iouType
        self.imgIds = list(imgIds)
        self.catIds = list(catIds)
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [1, 10, 100]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ["all", "small", "medium", "large"]
        self.useCats = 1


def summarize_eval(ev, params, out=print):
    """pycocotools' `COCOeval.summarize` for detections: the 12 lines through `out`, and the stats (12,)."""
    def one(ap=1, iouThr=None, areaRng="all", maxDets=100):
        p = params
        iStr = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}"
        titleStr = "Average Precision" if ap == 1 else "Average Recall"
        typeStr = "(AP)" if ap == 1 else "(AR)"
        iouStr = ("{:0.2f}:{:0.2f}".format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None
                  else "{:0.2f}".format(iouThr))
        aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
        mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
        if ap == 1:
            s = ev["precision"]
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, :, aind, mind]
        else:
            s = ev["recall"]
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, aind, mind]
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        out(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
        return mean_s

    m = params.maxDets
    stats = np.zeros((12,))
    stats[0] = one(1)
    stats[1] = one(1, iouThr=.5, maxDets=m[2])
    stats[2] = one(1, iouThr=.75, maxDets=m[2])
    stats[3] = one(1, areaRng="small", maxDets=m[2])
    stats[4] = one(1, areaRng="medium", maxDets=m[2])
    stats[5] = one(1, areaRng="large", maxDets=m[2])
    stats[6] = one(0, maxDets=m[0])
    stats[7] = one(0, maxDets=m[1])
    stats[8] = one(0, maxDets=m[2])
    stats[9] = one(0, areaRng="small", maxDets=m[2])
    stats[10] = one(0, areaRng="medium", maxDets=m[2])
    stats[11] = one(0, areaRng="large", maxDets=m[2])
    return stats


def load_dataset(coco_gt) -> dict:
    """The annotation dict of a COCO JSON path, a parsed dict, or an object with a `.dataset` dict (pycocotools'
    `COCO`, what `get_coco_api_from_dataset` returns)."""
    if isinstance(coco_gt, (str, os.PathLike)):
        with open(coco_gt) as f:
            return json.load(f)
    if isinstance(coco_gt, dict):
        return coco_gt
    if isinstance(getattr(coco_gt, "dataset", None), dict):
        return coco_gt.dataset
    raise TypeError(f"CocoEvaluator: coco_gt must be a path, a dict or have a .dataset dict, got {type(coco_gt)}")


def _runs(ann, h, w):
    """Column-major (start, length) of the runs of ones of an RLE segmentation."""
    seg = ann.get("segmentation")
    if not isinstance(seg, dict):
        raise NotImplementedError(f"coco_eval: annotation {ann.get('id')} has a polygon (or no) segmentation; only "
                                  f"RLE ground-truth masks are supported")
    if [int(v) for v in seg["size"]] != [h, w]:
        raise ValueError(f"coco_eval: annotation {ann.get('id')}'s mask is {seg['size']}, its image {h}x{w}")
    counts = seg["counts"]
    cnts = np.asarray(counts, np.int64) if isinstance(counts, list) else mots.decode_counts(counts)
    if (cnts < 0).any() or cnts.sum() != h * w:
        raise ValueError(f"coco_eval: annotation {ann.get('id')}'s runs do not cover a {h}x{w} mask")
    starts = np.concatenate(([0], np.cumsum(cnts)[:-1]))
    ones = (np.arange(len(cnts)) % 2 == 1) & (cnts > 0)
    return np.stack((starts[ones], cnts[ones]), 1)


class GroundTruth:
    """The ground truth packed for the kernels (host numpy arrays; `upload` copies them to a device once).

    Rows are the annotations of each image in JSON order, stably sorted by category index within the image;
    `off[i] .. off[i + 1]` are image i's rows, images in the order of `dataset["images"]`.  Annotations of categories
    outside `cat_ids` are left out, as pycocotools' `getAnnIds(catIds=...)` leaves them out.  With `device`, the segm
    ground truth's polygon and box-list segmentations are rasterised in one call there and read back once; without
    it they raise NotImplementedError."""

    def __init__(self, dataset: dict, segm: bool, device=None):
        images = dataset.get("images", [])
        self.img_ids = np.asarray([int(im["id"]) for im in images], np.int64)
        self.row_of = {int(i): r for r, i in enumerate(self.img_ids)}
        self.height = np.asarray([int(im.get("height", 0)) for im in images], np.int64)
        self.width = np.asarray([int(im.get("width", 0)) for im in images], np.int64)
        anns = dataset.get("annotations", [])
        if "categories" in dataset:
            self.cat_ids = np.asarray(sorted(int(c["id"]) for c in dataset["categories"]), np.int64)
        else:
            self.cat_ids = np.unique(np.asarray([int(a["category_id"]) for a in anns], np.int64))
        if len(self.cat_ids) == 0:
            raise ValueError("coco_eval: the ground truth has no categories")
        per_img = [[] for _ in images]
        for a in anns:
            r = self.row_of.get(int(a["image_id"]))
            k = np.searchsorted(self.cat_ids, int(a["category_id"]))
            if r is None or k >= len(self.cat_ids) or self.cat_ids[k] != int(a["category_id"]):
                continue
            per_img[r].append((int(k), a))
        rows = []
        self.off = np.zeros(len(images) + 1, np.int64)
        for r, lst in enumerate(per_img):
            lst.sort(key=lambda ka: ka[0])                   # stable: JSON order within a category
            ks = np.asarray([k for k, _ in lst], np.int64)
            if len(ks) and np.bincount(ks).max() > MAX_GT_PER_IMAGE_CATEGORY:
                raise ValueError(f"coco_eval: image {self.img_ids[r]} has more than {MAX_GT_PER_IMAGE_CATEGORY} "
                                 f"ground truths of one category")
            rows.extend((r, k, a) for k, a in lst)
            self.off[r + 1] = len(rows)
        n = len(rows)
        self.img_row = np.asarray([r for r, _, _ in rows], np.int64)
        self.k = np.asarray([k for _, k, _ in rows], np.int32)
        self.box = np.zeros((n, 4), np.float64)
        self.area = np.zeros(n, np.float64)
        self.crowd = np.zeros(n, np.uint8)
        self.id = np.zeros(n, np.int64)
        for i, (_, _, a) in enumerate(rows):
            if "area" not in a:
                raise ValueError(f"coco_eval: annotation {a.get('id')} has no area")
            if "bbox" in a:
                self.box[i] = np.asarray(a["bbox"], np.float64)
            self.area[i] = float(a["area"])
            self.crowd[i] = 1 if a.get("iscrowd", 0) else 0      # pycocotools' _prepare: ignore = iscrowd
            self.id[i] = int(a["id"])
        self.segm = segm
        if segm:
            self.bbox = np.zeros((n, 4), np.int32)
            self.px = np.zeros(n, np.int64)
            runs = []
            self.run_off = np.zeros(n + 1, np.int64)
            poly = {}
            if device is not None:
                rows_p = [i for i, (_, _, a) in enumerate(rows) if isinstance(a.get("segmentation"), list)]
                for i in rows_p:
                    r = rows[i][0]
                    if int(self.height[r]) * int(self.width[r]) >= 2 ** 31:
                        raise ValueError(f"coco_eval: image {self.img_ids[r]} is over 2^31 pixels")
                if rows_p:
                    p_off, p_runs = coco_masks.poly_runs(
                        [rows[i][2]["segmentation"] for i in rows_p],
                        [(int(self.height[rows[i][0]]), int(self.width[rows[i][0]])) for i in rows_p],
                        [f"annotation {rows[i][2].get('id')}" for i in rows_p], device)
                    poly = {i: p_runs[p_off[j]:p_off[j + 1]] for j, i in enumerate(rows_p)}
            for i, (r, _, a) in enumerate(rows):
                h, w = int(self.height[r]), int(self.width[r])
                if h * w >= 2 ** 31:
                    raise ValueError(f"coco_eval: image {self.img_ids[r]} is over 2^31 pixels")
                ru = poly[i] if i in poly else _runs(a, h, w)
                runs.append(ru)
                self.run_off[i + 1] = self.run_off[i] + len(ru)
                self.px[i] = int(ru[:, 1].sum()) if len(ru) else 0
                if len(ru):
                    last = ru[:, 0] + ru[:, 1] - 1
                    x0, x1 = int((ru[:, 0] // h).min()), int((last // h).max())
                    if ((ru[:, 0] // h) != (last // h)).any():
                        y0, y1 = 0, h - 1
                    else:
                        y0, y1 = int((ru[:, 0] % h).min()), int((last % h).max())
                    self.bbox[i] = (x0, y0, x1, y1)
                else:
                    self.bbox[i] = (1, 1, 0, 0)
            self.runs = (np.concatenate(runs) if runs else np.zeros((0, 2), np.int64)).astype(np.uint32)
        self._dev = {}

    def not_ignored(self, area_rng):
        """bool [rows, A]: the row counts towards npig in area range a (evaluateImg's gtIgnore == 0)."""
        lo, hi = np.asarray(area_rng, np.float64).T
        return (self.crowd[:, None] == 0) & ~(self.area[:, None] < lo) & ~(self.area[:, None] > hi)

    def npig(self, img_rows, area_rng):
        """int64 [K, A] non-ignored ground truths of the given images (pycocotools' npig)."""
        keep = np.zeros(len(self.img_ids), bool)
        keep[np.asarray(img_rows, np.int64)] = True
        sel = keep[self.img_row]
        ni = self.not_ignored(area_rng)[sel]
        K, A = len(self.cat_ids), len(area_rng)
        out = np.zeros((K, A), np.int64)
        for a in range(A):
            out[:, a] = np.bincount(self.k[sel][ni[:, a]], minlength=K)
        return out

    def arrays(self):
        a = dict(cat_ids=self.cat_ids, off=self.off, k=self.k, box=self.box, area=self.area, crowd=self.crowd,
                 id=self.id)
        if self.segm:
            a.update(run_off=self.run_off, runs=self.runs, bbox=self.bbox, px=self.px)
        return a

    def upload(self, device):
        key = str(device)
        if key not in self._dev:
            self._dev[key] = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in self.arrays().items()}
        return self._dev[key]


def kept_images(records):
    """The reference's `merge` on host records: `records` is a list of (image ids, detection counts) in rank order,
    then update order.  Returns (sorted unique image ids, first row of each in the concatenated records, its count):
    the first occurrence of every image id is kept, as `np.unique(..., return_index=True)` keeps it."""
    ids, begins, counts = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    base = 0
    for img_ids, cnt in records:
        cnt = np.asarray(cnt, np.int64)
        ids.append(np.asarray(img_ids, np.int64))
        begins.append(base + np.concatenate(([0], np.cumsum(cnt)[:-1])).astype(np.int64))
        counts.append(cnt)
        base += int(cnt.sum())
    ids, begins, counts = np.concatenate(ids), np.concatenate(begins), np.concatenate(counts)
    uniq, idx = np.unique(ids, return_index=True)
    return uniq, begins[idx], counts[idx]


def pack_update(gt, params, img_ids, predictions, segm):
    """Host side of one update: the image table and the detection tensors, on their given device.  Validates the
    predictions (ValueError).  Returns dict(img [B, 10] int64 numpy, boxes, scores, labels, masks, sizes)."""
    B = len(img_ids)
    img = np.zeros((B, _IMG_FIELDS), np.int64)
    boxes, scores, labels, masks = [], [], [], []
    n_at = iou_at = dbit_at = gbit_at = gtm_at = 0
    A, T = len(params.areaRng), len(params.iouThrs)
    max_n = max_g = 0
    for b, i in enumerate(img_ids):
        r = gt.row_of.get(int(i))
        if r is None:
            raise ValueError(f"coco_eval: image id {i} is not in the ground truth")
        pred = predictions[i]
        s = pred["scores"]
        n = int(s.shape[0]) if s.dim() else 0
        if s.dim() != 1 or s.dtype != torch.float32:
            raise ValueError(f"coco_eval: image {i}: scores must be a 1-D float32 tensor")
        if n > MAX_DETS_PER_IMAGE:
            raise ValueError(f"coco_eval: image {i} has {n} detections, over the limit of {MAX_DETS_PER_IMAGE}")
        if s.device.type == "cpu" and not torch.isfinite(s).all():
            raise ValueError(f"coco_eval: image {i} has a non-finite score")
        lab = pred["labels"]
        if tuple(lab.shape) != (n,):
            raise ValueError(f"coco_eval: image {i}: labels must have shape ({n},)")
        scores.append(s)
        labels.append(lab)
        if segm:
            m = pred["masks"]
            h, w = int(gt.height[r]), int(gt.width[r])
            if m.dim() != 4 or tuple(m.shape) != (n, 1, h, w):
                raise ValueError(f"coco_eval: image {i}: masks must be [{n}, 1, {h}, {w}], got {tuple(m.shape)}")
            if m.dtype not in (torch.bool, torch.uint8):     # the kernel reads one byte per pixel, nonzero = set
                m = m > 0.5                                    # what the reference's `masks > 0.5` keeps
            masks.append(m.contiguous())
            plane = w * ((h + 31) // 32)
            img[b, 3], img[b, 4] = h, w
        else:
            bx = pred["boxes"]
            if tuple(bx.shape) != (n, 4) or bx.dtype != torch.float32:
                raise ValueError(f"coco_eval: image {i}: boxes must be a [{n}, 4] float32 tensor")
            boxes.append(bx)
            plane = 0
        g = int(gt.off[r + 1] - gt.off[r])
        img[b, 0], img[b, 1], img[b, 2] = r, n_at, n
        img[b, 6], img[b, 7], img[b, 8], img[b, 9] = iou_at, dbit_at, gbit_at, gtm_at
        n_at += n
        iou_at += n * g
        dbit_at += n * plane
        gbit_at += g * plane
        gtm_at += A * T * g
        max_n, max_g = max(max_n, n), max(max_g, g)
    return dict(img=img, boxes=boxes, scores=scores, labels=labels, masks=masks, N=n_at, iou_cells=iou_at,
                dbit_words=dbit_at, gbit_words=gbit_at, gtm_bytes=gtm_at, max_n=max_n, max_g=max_g)


def eval_dict(params, precision, recall, scores):
    T, R, K, A, M = precision.shape
    return {"params": params, "counts": [T, R, K, A, M],
            "date": datetime.datetime.now().strftime("%Y-%m-%d %H:%M:%S"),
            "precision": precision, "recall": recall, "scores": scores}


_lib = None


def _library():
    global _lib
    if _lib is None:
        from . import ext
        ext.load()                                   # raises with the build command when the native code is missing
        lib = ctypes.CDLL(ext.library_path())
        vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t
        lib.tfb200_coco_match_workspace_bytes.argtypes = [i64] * 5
        lib.tfb200_coco_match_workspace_bytes.restype = sz
        lib.tfb200_coco_match_f32.argtypes = ([vp, i32, i32, i32, vp, vp, vp, i64, vp, i32] + [vp] * 11
                                              + [i32, vp, i32, i32, i32, i64, i64, i64, i64, vp, sz, vp, vp, vp, vp,
                                                 vp])
        lib.tfb200_coco_match_f32.restype = i32
        lib.tfb200_coco_accumulate_workspace_bytes.argtypes = [i64]
        lib.tfb200_coco_accumulate_workspace_bytes.restype = sz
        lib.tfb200_coco_accumulate_f32.argtypes = ([vp, vp, vp, i64, vp, i32, i64, vp, vp, vp, vp, i32, i32, i32, i32,
                                                    i32, vp, sz, vp, vp, vp, vp, vp])
        lib.tfb200_coco_accumulate_f32.restype = i32
        _lib = lib
    return _lib


_DUMMY = {}


def _ptr(t):
    """A tensor's address; an empty tensor gets a valid one that is never read (the C entries reject NULL)."""
    if t is None:
        return None
    if t.numel():
        return t.data_ptr()
    if t.device not in _DUMMY:
        _DUMMY[t.device] = torch.zeros(64, dtype=torch.float64, device=t.device)
    return _DUMMY[t.device].data_ptr()


class _Records:
    """One update's (or one rank's) per-detection records: image ids and detection counts on the host; key, rank and
    state on the device (or host numpy arrays after a gather across ranks)."""

    def __init__(self, img_ids, counts, key, rank, state):
        self.img_ids, self.counts, self.key, self.rank, self.state = img_ids, counts, key, rank, state

    def to_host(self):
        return _Records(self.img_ids, self.counts, *(x.cpu().numpy() if torch.is_tensor(x) else x
                                                     for x in (self.key, self.rank, self.state)))


class COCOevalGPU:
    """What the reference reads of pycocotools' `COCOeval`: `params`, `eval`, `stats` and `summarize()`."""

    def __init__(self, iou_type, cat_ids):
        self.params = Params(iou_type, cat_ids)
        self.eval = {}
        self.stats = []

    def summarize(self):
        if not self.eval:
            raise Exception("Please run accumulate() first")
        self.stats = summarize_eval(self.eval, self.params)

    def __str__(self):
        self.summarize()
        return ""


class CocoEvaluator:
    """Drop-in for the reference's `CocoEvaluator` (datasets/coco_eval.py): `update`, `synchronize_between_processes`,
    `accumulate`, `summarize`, and `coco_eval[iou_type]` with `.params`, `.eval`, `.stats`, `.summarize()`."""

    def __init__(self, coco_gt, iou_types, device=None):
        if not isinstance(iou_types, (list, tuple)) or any(t not in IOU_TYPES for t in iou_types):
            raise ValueError(f"CocoEvaluator: iou_types must be a list or tuple from {IOU_TYPES}, got {iou_types!r}")
        if not torch.cuda.is_available():
            raise RuntimeError("coco_eval needs a CUDA device: the evaluation runs on the GPU and has no host fallback")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.coco_gt = coco_gt
        self.iou_types = tuple(iou_types)
        dataset = load_dataset(coco_gt)
        self.gt = {t: GroundTruth(dataset, t == "segm", self.device if t == "segm" else None) for t in self.iou_types}
        self.coco_eval = {t: COCOevalGPU(t, self.gt[t].cat_ids.tolist()) for t in self.iou_types}
        self.img_ids = []
        self._records = {t: [] for t in self.iou_types}
        self._status = {t: torch.zeros(1, dtype=torch.int32, device=self.device) for t in self.iou_types}
        self._kept = {}
        p = self.coco_eval[self.iou_types[0]].params if self.iou_types else Params()
        self._consts = {
            "area_rng": torch.tensor(np.asarray(p.areaRng, np.float64), device=self.device),
            "iou_thr": torch.tensor(np.minimum(p.iouThrs, 1 - 1e-10), device=self.device),
            "rec_thr": torch.tensor(p.recThrs, device=self.device),
            "max_dets": torch.tensor(np.asarray(p.maxDets, np.int32), device=self.device)}

    def update(self, predictions):
        img_ids = [int(i) for i in np.unique(np.asarray(list(predictions.keys()), np.int64))]
        if not img_ids:
            return
        self.img_ids.extend(img_ids)
        self._kept = {}
        for t in self.iou_types:
            self._records[t].append(self._match(t, img_ids, predictions))

    def _match(self, iou_type, img_ids, predictions):
        gt, params, dev = self.gt[iou_type], self.coco_eval[iou_type].params, self.device
        segm = iou_type == "segm"
        z = pack_update(gt, params, img_ids, predictions, segm)
        g = gt.upload(dev)
        A, T = len(params.areaRng), len(params.iouThrs)
        N = z["N"]
        img = z["img"]
        if segm:
            masks = [m.to(dev, non_blocking=True) for m in z["masks"]]
            img[:, 5] = [m.data_ptr() for m in masks]
        img_dev = torch.from_numpy(img).pin_memory().to(dev, non_blocking=True)
        cat = lambda xs, dt: (torch.cat([x.to(dev, dt, non_blocking=True) for x in xs]) if xs
                              else torch.zeros(0, dtype=dt, device=dev))
        scores, labels = cat(z["scores"], torch.float32), cat(z["labels"], torch.int64)
        boxes = None if segm else cat(z["boxes"], torch.float32).contiguous()
        key = torch.empty(N, dtype=torch.int64, device=dev)
        rank = torch.empty(N, dtype=torch.int32, device=dev)
        state = torch.empty(N * A, dtype=torch.int32, device=dev)
        lib = _library()
        sizes = (N, z["iou_cells"], z["dbit_words"], z["gbit_words"], z["gtm_bytes"])
        ws_bytes = lib.tfb200_coco_match_workspace_bytes(*sizes)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        rc = lib.tfb200_coco_match_f32(
            img_dev.data_ptr(), len(img_ids), z["max_n"], z["max_g"], _ptr(boxes), _ptr(scores), _ptr(labels), N,
            g["cat_ids"].data_ptr(), len(gt.cat_ids), g["off"].data_ptr(), _ptr(g["k"]), _ptr(g["box"]),
            _ptr(g["area"]), _ptr(g["crowd"]), _ptr(g["id"]), _ptr(g.get("run_off")), _ptr(g.get("runs")),
            _ptr(g.get("bbox")), _ptr(g.get("px")), self._consts["area_rng"].data_ptr(), A,
            self._consts["iou_thr"].data_ptr(), T, params.maxDets[-1], int(segm), *sizes[1:], ws.data_ptr(),
            ws_bytes, _ptr(key), _ptr(rank), _ptr(state), self._status[iou_type].data_ptr(), stream)
        if rc != 0:
            raise RuntimeError(f"tfb200_coco_match_f32 failed (code {rc})")
        counts = np.asarray([int(s.shape[0]) for s in z["scores"]], np.int64)
        return _Records(np.asarray(img_ids, np.int64), counts, key, rank, state)

    def synchronize_between_processes(self):
        import torch.distributed as dist
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        for t in self.iou_types:
            recs = self._records[t]
            if world > 1:
                local = ([r.to_host() for r in recs], int(self._status[t].item()))
                gathered = [None] * world
                dist.all_gather_object(gathered, local)
                recs = [r for rank_recs, _ in gathered for r in rank_recs]
                status = 0
                for _, s in gathered:
                    status |= s
                self._records[t] = recs
                self._status[t].fill_(status)
            self._kept[t] = kept_images([(r.img_ids, r.counts) for r in recs])

    def accumulate(self):
        for t in self.iou_types:
            self._accumulate(t)

    def _accumulate(self, iou_type):
        gt, ce, dev = self.gt[iou_type], self.coco_eval[iou_type], self.device
        p = ce.params
        recs = self._records[iou_type]
        ids, begins, counts = self._kept.get(iou_type) or kept_images([(r.img_ids, r.counts) for r in recs])
        p.imgIds = ids.tolist()
        K, A, T, R, M = len(gt.cat_ids), len(p.areaRng), len(p.iouThrs), len(p.recThrs), len(p.maxDets)
        as_dev = lambda x: x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x)).to(dev)
        key = torch.cat([as_dev(r.key) for r in recs]) if recs else torch.zeros(0, dtype=torch.int64, device=dev)
        rank = torch.cat([as_dev(r.rank) for r in recs]) if recs else torch.zeros(0, dtype=torch.int32, device=dev)
        state = torch.cat([as_dev(r.state) for r in recs]) if recs else torch.zeros(0, dtype=torch.int32, device=dev)
        dst = np.concatenate(([0], np.cumsum(counts)[:-1])).astype(np.int64)
        n = int(counts.sum())
        kept = torch.from_numpy(np.stack((begins, dst, counts), 1).astype(np.int64).reshape(-1, 3)).to(dev)
        npig = torch.from_numpy(gt.npig([gt.row_of[i] for i in p.imgIds], p.areaRng)).to(dev)
        out = torch.empty(2 * T * R * K * A * M + T * K * A * M + 1, dtype=torch.float64, device=dev)
        n5, n4 = T * R * K * A * M, T * K * A * M
        lib = _library()
        ws_bytes = lib.tfb200_coco_accumulate_workspace_bytes(n)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        base = out.data_ptr()
        rc = lib.tfb200_coco_accumulate_f32(
            _ptr(key), _ptr(rank), _ptr(state), key.numel(), kept.data_ptr(), len(ids), n, npig.data_ptr(),
            self._consts["rec_thr"].data_ptr(), self._consts["max_dets"].data_ptr(), self._status[iou_type].data_ptr(),
            K, A, T, R, M, ws.data_ptr(), ws_bytes, base, base + 8 * n5, base + 8 * (n5 + n4),
            base + 8 * (2 * n5 + n4), torch.cuda.current_stream(dev).cuda_stream)
        if rc != 0:
            raise RuntimeError(f"tfb200_coco_accumulate_f32 failed (code {rc})")
        host = out.cpu().numpy()                               # the one read-back
        if int(host[-1]) & 1:
            raise ValueError("coco_eval: an update had a non-finite score")
        precision = host[:n5].reshape(T, R, K, A, M).copy()
        recall = host[n5:n5 + n4].reshape(T, K, A, M).copy()
        scores = host[n5 + n4:2 * n5 + n4].reshape(T, R, K, A, M).copy()
        ce.eval = eval_dict(copy.deepcopy(p), precision, recall, scores)

    def summarize(self):
        for iou_type, coco_eval in self.coco_eval.items():
            print(f"IoU metric: {iou_type}")
            coco_eval.summarize()
