"""Panoptic quality (PQ) on the GPU, in place of the reference's `PanopticEvaluator`
(src/trackformer/datasets/panoptic_eval.py), which scores a panoptic model with panopticapi's `pq_compute`
(`engine.evaluate` reports its All / Things / Stuff dicts as `PQ_all`, `PQ_th`, `PQ_st`).

`PanopticEvaluator(ann_file, ann_folder, output_dir)` has the reference's methods.  `update(predictions)` writes each
prediction's PNG as the reference does and enqueues its scoring (csrc/panoptic.cu) without synchronising: the
image's ground-truth PNG is decoded on the host and uploaded, and the prediction map is the post-processor's device
`label_map` when `PostProcessPanoptic(maps_on_device=True)` made one (no PNG decode), else the decoded PNG.
`summarize()` writes `predictions.json` and returns `pq_compute`'s dict after one reduction launch and one read-back.
`pq_compute(gt_json_file, pred_json_file, gt_folder, pred_folder)` scores exported results from PNG folders.

The numbers are panopticapi's:
  * OFFSET = 2^24 and VOID = 0; ids are `rgb2id` of the PNGs (R + 256 G + 256^2 B).
  * GT segment areas are the JSON `area`, not recounted; prediction areas are counted from the PNG.
  * A (GT, prediction) pair is skipped for a crowd GT, a GT id not listed in the JSON, and different categories;
    otherwise union = pred_area + gt_area - intersection - |VOID ∩ pred|, and IoU > 0.5 is a match (tp, IoU summed).
  * An unmatched crowd GT is recorded per category (the last one in JSON order wins) and is not a false negative;
    every other unmatched GT is one.
  * An unmatched prediction is not a false positive when (|VOID ∩ p| + |crowd(cat) ∩ p|) / pred_area > 0.5.
  * `pq_average` skips categories with tp + fp + fn = 0, for All, Things and Stuff, and adds `per_class` under All.
  * Errors, with panopticapi's exception types and messages: a prediction id in the PNG but not in the JSON and a
    present segment of an unknown category (KeyError, the smaller id first), an id in the JSON but not in the PNG
    (KeyError), a GT image without a prediction (Exception).  Predictions with the same `image_id` resolve to the last
    one.  A prediction map whose size differs from the GT's raises ValueError.
The per-image IoU sums are added in ascending GT id and then over images in GT JSON order, in fp64; counts are exact,
so results repeat bit for bit.  Limits: TFB200_PANOPTIC_MAX_SEGMENTS (1024) listed segments per image and side, 4096
categories, fewer than 2^31 pixels per image; beyond them ValueError, nothing is truncated.  CUDA only.
"""
from __future__ import annotations

import ctypes
import io
import json
import os

import numpy as np
import torch
from PIL import Image

__all__ = ["PanopticEvaluator", "pq_compute", "id2rgb", "rgb2id", "MAX_SEGMENTS", "MAX_CATEGORIES", "MAX_KEPT"]

OFFSET = 256 * 256 * 256
VOID = 0
MAX_KEPT = 1024          # TFB200_PANOPTIC_MAX_KEPT (include/tfb200_fused.h)
MAX_SEGMENTS = 1024      # TFB200_PANOPTIC_MAX_SEGMENTS
MAX_CATEGORIES = 4096    # TFB200_PANOPTIC_MAX_CATEGORIES
BLOCK_PIXELS = 4096      # kBlockPixels (csrc/panoptic_core.h)
_PQ_FIELDS = 10
_LLMAX = np.iinfo(np.int64).max


def id2rgb(id_map):
    """panopticapi.utils.id2rgb: an id map -> uint8 RGB (R + 256 G + 256^2 B); a scalar id -> [r, g, b]."""
    if isinstance(id_map, np.ndarray):
        id_map_copy = id_map.copy()
        rgb_shape = tuple(list(id_map.shape) + [3])
        rgb_map = np.zeros(rgb_shape, dtype=np.uint8)
        for i in range(3):
            rgb_map[..., i] = id_map_copy % 256
            id_map_copy //= 256
        return rgb_map
    color = []
    for _ in range(3):
        color.append(id_map % 256)
        id_map //= 256
    return color


def rgb2id(color):
    """panopticapi.utils.rgb2id: uint8 RGB -> int32 ids (an array), or a scalar id from [r, g, b]."""
    if isinstance(color, np.ndarray) and len(color.shape) == 3:
        if color.dtype == np.uint8:
            color = color.astype(np.int32)
        return color[:, :, 0] + 256 * color[:, :, 1] + 256 * 256 * color[:, :, 2]
    return int(color[0] + 256 * color[1] + 256 * 256 * color[2])


def png_of(id_map: np.ndarray) -> bytes:
    """Pillow's PNG of `id2rgb(id_map)`: the post-processor's `png_string`."""
    with io.BytesIO() as out:
        Image.fromarray(id2rgb(id_map)).save(out, format="PNG")
        return out.getvalue()


def read_png_ids(path) -> np.ndarray:
    return rgb2id(np.array(Image.open(path), dtype=np.uint32)).astype(np.int32)


_lib = None


def _library():
    global _lib
    if _lib is None:
        from . import ext
        ext.load()                                   # raises with the build command when the native code is missing
        _lib = bind(ctypes.CDLL(ext.library_path()))
    return _lib


def bind(lib):
    """Declares the panoptic C entries' arguments on a ctypes library (the product's, or a test's host build of the
    same routines under the same names)."""
    vp, i32, i64, f32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
    lib.tfb200_panoptic_classes_f32.argtypes = [vp, i32, i32, i32, f32, vp, vp, vp, vp]
    lib.tfb200_panoptic_label_f32.argtypes = [vp, i32, i32, i32, i32, vp, i32, vp, vp, vp, vp, vp, vp, i32, vp]
    lib.tfb200_panoptic_final_f32.argtypes = [vp, i32, vp, vp, vp, vp, vp, i32, vp]
    lib.tfb200_pq_update.argtypes = [vp, i32, i32, i32] + [vp] * 9 + [i64] + [vp] * 4 + [i32, vp]
    lib.tfb200_pq_reduce.argtypes = [vp, vp, vp, vp, i64, i32, vp, vp, vp]
    for f in ("tfb200_panoptic_classes_f32", "tfb200_panoptic_label_f32", "tfb200_panoptic_final_f32",
              "tfb200_pq_update", "tfb200_pq_reduce"):
        getattr(lib, f).restype = i32
    return lib


def check(rc, name):
    if rc != 0:
        raise RuntimeError(f"{name} failed (code {rc})")


def stream_of(device):
    return torch.cuda.current_stream(device).cuda_stream if device.type == "cuda" else None


# ---------------------------------------------------------------------------------------------------------------------
class Categories:
    """`gt_json["categories"]` in JSON order: category id -> dense index, and the thing flags."""

    def __init__(self, categories):
        self.ids = [int(c["id"]) for c in categories]
        self.items = {int(c["id"]): c for c in categories}
        if len(self.ids) > MAX_CATEGORIES:
            raise ValueError(f"panoptic_eval: {len(self.ids)} categories, over the limit of {MAX_CATEGORIES}")
        if not self.ids:
            raise ValueError("panoptic_eval: the ground truth has no categories")
        self.index = {c: k for k, c in enumerate(self.ids)}


class PQScorer:
    """Per-image PQ records on one device.  `add(items)` enqueues one batch of images, each a dict with `gt_ann`,
    `gt_map` (int32 [H, W] raw ids, numpy or tensor), `pred_ann` and `pred_map` (raw ids, numpy or tensor); `result(
    image_ids)` reduces the records of the given images (the last record of each id) in that order."""

    def __init__(self, categories, device, lib=None):
        self.lib = lib or _library()
        self.cats = Categories(categories)
        self.device = torch.device(device)
        Kc = len(self.cats.ids)
        self.Kc = Kc
        self._stat_i, self._stat_iou, self._err, self._pred_area = [], [], [], []
        self._row_of = {}            # image id -> global record row (the last update wins)
        self._rows = 0
        self._batches = []           # (first row, per-image prediction info) for error messages

    def add(self, items):
        if not items:
            return
        dev, Kc = self.device, self.Kc
        B = len(items)
        img = np.zeros((B, _PQ_FIELDS), np.int64)
        gt_tabs, pred_tabs, maps = [], [], []
        go = po = mo = co = 0
        max_pix = max_seg = 0
        infos = []
        for b, it in enumerate(items):
            gt_ann, pred_ann = it["gt_ann"], it["pred_ann"]
            gmap, pmap = it["gt_map"], it["pred_map"]
            if tuple(gmap.shape) != tuple(pmap.shape):
                raise ValueError(f"panoptic_eval: image {gt_ann['image_id']}: the prediction map is "
                                 f"{tuple(pmap.shape)}, the ground truth {tuple(gmap.shape)}")
            npix = int(np.prod(gmap.shape))
            if npix >= 2 ** 31:
                raise ValueError(f"panoptic_eval: image {gt_ann['image_id']} has 2^31 pixels or more")
            gsegs = {int(el["id"]): el for el in gt_ann["segments_info"]}       # panopticapi's dicts
            psegs = {int(el["id"]): el for el in pred_ann["segments_info"]}
            G, P = len(gsegs), len(psegs)
            if G > MAX_SEGMENTS or P > MAX_SEGMENTS:
                raise ValueError(f"panoptic_eval: image {gt_ann['image_id']} has {max(G, P)} segments, over the "
                                 f"limit of {MAX_SEGMENTS}")
            json_pos = {k: i for i, k in enumerate(gsegs)}
            gid = sorted(gsegs)
            pid = sorted(psegs)
            gt_tabs.append((np.asarray(gid, np.int32),
                            np.asarray([self.cats.index.get(int(gsegs[i]["category_id"]), -1) for i in gid], np.int32),
                            np.asarray([1 if gsegs[i].get("iscrowd", 0) == 1 else 0 for i in gid], np.int32),
                            np.asarray([gsegs[i]["area"] for i in gid], np.float64),
                            np.asarray([json_pos[i] for i in gid], np.int32)))
            pred_tabs.append((np.asarray(pid, np.int32),
                              np.asarray([self.cats.index.get(int(psegs[i]["category_id"]), -1) for i in pid],
                                         np.int32)))
            infos.append((gt_ann["image_id"], pid, [psegs[i]["category_id"] for i in pid]))
            maps.append((gmap, pmap))
            img[b] = (npix, mo, mo + npix, go, G, gid.index(0) if 0 in gsegs else G, po, P, co, b)
            mo += 2 * npix
            go += G
            po += P
            co += (G + 2) * (P + 1)
            max_pix, max_seg = max(max_pix, npix), max(max_seg, G, P)
        flat = torch.empty(mo, dtype=torch.int32, device=dev)
        for b, (gmap, pmap) in enumerate(maps):
            o, n = int(img[b, 1]), int(img[b, 0])
            for dst, m in ((flat[o:o + n], gmap), (flat[o + n:o + 2 * n], pmap)):
                m = torch.as_tensor(m) if isinstance(m, np.ndarray) else m
                dst.copy_(m.reshape(-1).to(dtype=torch.int32), non_blocking=True)
        cat = lambda arrs, dt: np.ascontiguousarray(np.concatenate(arrs).astype(dt) if arrs else np.zeros(0, dt))
        host = [cat([t[i] for t in gt_tabs], dt) for i, dt in enumerate((np.int32, np.int32, np.int32, np.float64,
                                                                          np.int32))]
        host += [cat([t[i] for t in pred_tabs], np.int32) for i in range(2)]
        up = lambda a: torch.from_numpy(a if a.size else np.zeros(1, a.dtype)).to(dev, non_blocking=True)
        gt_id, gt_cat, gt_crowd, gt_area, gt_json, pred_id, pred_cat = (up(a) for a in host)
        img_dev = up(img)
        cells = torch.empty(max(co, 1), dtype=torch.int32, device=dev)
        pred_area = torch.empty(max(po, 1), dtype=torch.int64, device=dev)
        stat_i = torch.empty((B, Kc, 3), dtype=torch.int32, device=dev)
        stat_iou = torch.empty((B, Kc), dtype=torch.float64, device=dev)
        err = torch.tensor([[_LLMAX, _LLMAX, 0]] * B, dtype=torch.int64).to(dev, non_blocking=True)
        blocks = max(1, (max_pix + BLOCK_PIXELS - 1) // BLOCK_PIXELS)
        rc = self.lib.tfb200_pq_update(
            img_dev.data_ptr(), B, Kc, max_seg, flat.data_ptr(), gt_id.data_ptr(), gt_cat.data_ptr(),
            gt_crowd.data_ptr(), gt_area.data_ptr(), gt_json.data_ptr(), pred_id.data_ptr(), pred_cat.data_ptr(),
            cells.data_ptr(), cells.numel(), pred_area.data_ptr(), stat_i.data_ptr(), stat_iou.data_ptr(),
            err.data_ptr(), blocks, stream_of(dev))
        check(rc, "tfb200_pq_update")
        self._stat_i.append(stat_i)
        self._stat_iou.append(stat_iou)
        self._err.append(err)
        self._pred_area.append((pred_area, img[:, 6].copy(), img[:, 7].copy()))
        for b, it in enumerate(items):
            self._row_of[int(it["gt_ann"]["image_id"])] = self._rows + b
        self._batches.append((self._rows, infos))
        self._rows += B

    def result(self, image_ids):
        """(per-category tp, fp, fn, iou as numpy arrays in category order) over the given images, raising
        panopticapi's errors (the first image in the given order that has one)."""
        dev, Kc = self.device, self.Kc
        for i in image_ids:
            if int(i) not in self._row_of:
                raise Exception('no prediction for the image with id: {}'.format(i))
        rows = torch.from_numpy(np.asarray([self._row_of[int(i)] for i in image_ids], np.int64)).to(dev)
        if self._stat_i:
            stat_i, stat_iou, err = torch.cat(self._stat_i), torch.cat(self._stat_iou), torch.cat(self._err)
        else:
            stat_i = torch.zeros((1, Kc, 3), dtype=torch.int32, device=dev)
            stat_iou = torch.zeros((1, Kc), dtype=torch.float64, device=dev)
            err = torch.zeros((1, 3), dtype=torch.int64, device=dev)
        out = torch.empty(Kc * 4 + 1, dtype=torch.float64, device=dev)
        err_out = out[Kc * 4:].view(torch.int64)
        rc = self.lib.tfb200_pq_reduce(stat_i.data_ptr(), stat_iou.data_ptr(), err.data_ptr(),
                                         rows.data_ptr() if rows.numel() else out.data_ptr(), rows.numel(), Kc,
                                         out.data_ptr(), err_out.data_ptr(), stream_of(dev))
        check(rc, "tfb200_pq_reduce")
        host = out.cpu().numpy()                                    # the one read-back
        first = int(host[Kc * 4:].view(np.int64)[0])
        if first < len(image_ids):
            self._raise(self._row_of[int(image_ids[first])], err)
        s = host[:Kc * 4].reshape(Kc, 4)
        return s[:, 0].astype(np.int64), s[:, 1].astype(np.int64), s[:, 2].astype(np.int64), s[:, 3].copy()

    def _raise(self, row, err):
        e = err[row].cpu().numpy()
        for first, infos in reversed(self._batches):
            if row >= first:
                image_id, pid, pcat = infos[row - first]
                b = row - first
                break
        unlisted, unknown, missing = int(e[0]), int(e[1]), int(e[2])
        if unlisted != _LLMAX and unlisted < unknown:
            raise KeyError('In the image with ID {} segment with ID {} is presented in PNG and not presented in '
                           'JSON.'.format(image_id, unlisted))
        if unknown != _LLMAX:
            raise KeyError('In the image with ID {} segment with ID {} has unknown category_id {}.'.format(
                image_id, unknown, pcat[pid.index(unknown)]))
        bi = next(i for i, (f, _) in enumerate(self._batches) if f == first)
        area_t, offs, counts = self._pred_area[bi]
        areas = area_t[int(offs[b]):int(offs[b]) + int(counts[b])].cpu().numpy()
        absent = [pid[j] for j in range(len(pid)) if areas[j] == 0]
        raise KeyError('In the image with ID {} the following segment IDs {} are presented in JSON and not presented '
                       'in PNG.'.format(image_id, absent))


def pq_results(cats: Categories, tp, fp, fn, iou):
    """panopticapi's `pq_average` for All, Things and Stuff (`per_class` under All)."""
    results = {}
    for name, isthing in (("All", None), ("Things", True), ("Stuff", False)):
        pq, sq, rq, n = 0, 0, 0, 0
        per_class = {}
        for k, label in enumerate(cats.ids):
            if isthing is not None and isthing != (cats.items[label]["isthing"] == 1):
                continue
            t, f_p, f_n, io = int(tp[k]), int(fp[k]), int(fn[k]), float(iou[k])
            if t + f_p + f_n == 0:
                per_class[label] = {"pq": 0.0, "sq": 0.0, "rq": 0.0}
                continue
            n += 1
            pq_class = io / (t + 0.5 * f_p + 0.5 * f_n)
            sq_class = io / t if t != 0 else 0
            rq_class = t / (t + 0.5 * f_p + 0.5 * f_n)
            per_class[label] = {"pq": pq_class, "sq": sq_class, "rq": rq_class}
            pq += pq_class
            sq += sq_class
            rq += rq_class
        results[name] = {"pq": pq / n, "sq": sq / n, "rq": rq / n, "n": n}
        if name == "All":
            results["per_class"] = per_class
    return results


def print_table(results):
    print("{:10s}| {:>5s}  {:>5s}  {:>5s} {:>5s}".format("", "PQ", "SQ", "RQ", "N"))
    print("-" * (10 + 7 * 4))
    for name in ("All", "Things", "Stuff"):
        print("{:10s}| {:5.1f}  {:5.1f}  {:5.1f} {:5d}".format(
            name, 100 * results[name]["pq"], 100 * results[name]["sq"], 100 * results[name]["rq"],
            results[name]["n"]))


def _device(device):
    if device is not None:
        return torch.device(device)
    if not torch.cuda.is_available():
        raise RuntimeError("panoptic_eval needs a CUDA device: the scoring runs on the GPU and has no host fallback")
    return torch.device("cuda", torch.cuda.current_device())


def pq_compute(gt_json_file, pred_json_file, gt_folder=None, pred_folder=None, device=None, batch=16, lib=None):
    """panopticapi's `pq_compute` on the GPU: scores the PNG folders of exported results, prints the table and
    returns {"All", "Things", "Stuff": {"pq", "sq", "rq", "n"}, "per_class"}."""
    with open(gt_json_file) as f:
        gt_json = json.load(f)
    with open(pred_json_file) as f:
        pred_json = json.load(f)
    if gt_folder is None:
        gt_folder = gt_json_file.replace(".json", "")
    if pred_folder is None:
        pred_folder = pred_json_file.replace(".json", "")
    print("Evaluation panoptic segmentation metrics:")
    print("Ground truth:")
    print("\tSegmentation folder: {}".format(gt_folder))
    print("\tJSON file: {}".format(gt_json_file))
    print("Prediction:")
    print("\tSegmentation folder: {}".format(pred_folder))
    print("\tJSON file: {}".format(pred_json_file))
    if not os.path.isdir(gt_folder):
        raise Exception("Folder {} with ground truth segmentations doesn't exist".format(gt_folder))
    if not os.path.isdir(pred_folder):
        raise Exception("Folder {} with predicted segmentations doesn't exist".format(pred_folder))
    pred_annotations = {el["image_id"]: el for el in pred_json["annotations"]}
    for gt_ann in gt_json["annotations"]:
        if gt_ann["image_id"] not in pred_annotations:
            raise Exception("no prediction for the image with id: {}".format(gt_ann["image_id"]))
    scorer = PQScorer(gt_json["categories"], _device(device), lib)
    anns = gt_json["annotations"]
    for c in range(0, len(anns), batch):
        items = []
        for gt_ann in anns[c:c + batch]:
            pred_ann = pred_annotations[gt_ann["image_id"]]
            items.append(dict(gt_ann=gt_ann, pred_ann=pred_ann,
                              gt_map=read_png_ids(os.path.join(gt_folder, gt_ann["file_name"])),
                              pred_map=read_png_ids(os.path.join(pred_folder, pred_ann["file_name"]))))
        scorer.add(items)
    results = pq_results(scorer.cats, *scorer.result([a["image_id"] for a in anns]))
    print_table(results)
    return results


class PanopticEvaluator:
    """Drop-in for the reference's `PanopticEvaluator` (datasets/panoptic_eval.py): `update`,
    `synchronize_between_processes` and `summarize`, scored on the GPU."""

    def __init__(self, ann_file, ann_folder, output_dir="panoptic_eval", device=None, lib=None):
        self.gt_json = ann_file
        self.gt_folder = ann_folder
        if _is_main_process() and not os.path.exists(output_dir):
            os.mkdir(output_dir)
        self.output_dir = output_dir
        self.predictions = []
        with open(ann_file) as f:
            gt = json.load(f)
        self._gt_anns = gt["annotations"]
        self._gt_of = {a["image_id"]: a for a in self._gt_anns}
        self._scorer = PQScorer(gt["categories"], _device(device), lib)

    def update(self, predictions):
        items = []
        for p in predictions:
            png = p.pop("png_string")
            with open(os.path.join(self.output_dir, p["file_name"]), "wb") as f:
                f.write(png)
            label_map = p.pop("label_map", None)
            gt_ann = self._gt_of.get(p["image_id"])
            if gt_ann is None:                       # panopticapi scores the ground truth's images only
                continue
            pred_map = label_map if label_map is not None else rgb2id(np.array(Image.open(io.BytesIO(png)),
                                                                               dtype=np.uint32)).astype(np.int32)
            gt_map = read_png_ids(os.path.join(self.gt_folder, gt_ann["file_name"]))
            items.append(dict(gt_ann=gt_ann, pred_ann=p, gt_map=gt_map, pred_map=pred_map))
        self._scorer.add(items)
        self.predictions += predictions

    def synchronize_between_processes(self):
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise NotImplementedError("PanopticEvaluator: multi-process evaluation is not supported; the records "
                                      "stay on each rank's device")

    def summarize(self):
        if not _is_main_process():
            return None
        with open(os.path.join(self.output_dir, "predictions.json"), "w") as f:
            f.write(json.dumps({"annotations": self.predictions}, default=_json_default))
        ids = [a["image_id"] for a in self._gt_anns]
        results = pq_results(self._scorer.cats, *self._scorer.result(ids))
        print_table(results)
        return results


def _json_default(o):
    if isinstance(o, np.generic):
        return o.item()
    raise TypeError(f"{type(o)} is not JSON serializable")


def _is_main_process():
    import torch.distributed as dist
    return not (dist.is_available() and dist.is_initialized()) or dist.get_rank() == 0
