"""Numpy restatement of panopticapi's `pq_compute` (the oracle of the PQ tests): per image `np.unique` over the 64-bit
(GT id * 2^24 + prediction id) pixel keys, the match / FN / FP rules of `pq_compute_single_core`, and `pq_average`.
Images are scored sequentially in GT JSON order; errors carry panopticapi's types and messages."""
from collections import defaultdict

import numpy as np

OFFSET = 256 * 256 * 256
VOID = 0


class PQStatCat:
    def __init__(self):
        self.iou, self.tp, self.fp, self.fn = 0.0, 0, 0, 0


def score_image(stat, gt_ann, pan_gt, pred_ann, pan_pred, categories):
    gt_segms = {el["id"]: dict(el) for el in gt_ann["segments_info"]}
    pred_segms = {el["id"]: dict(el) for el in pred_ann["segments_info"]}
    pred_labels_set = set(el["id"] for el in pred_ann["segments_info"])
    labels, labels_cnt = np.unique(pan_pred, return_counts=True)
    for label, label_cnt in zip(labels, labels_cnt):
        label = int(label)
        if label not in pred_segms:
            if label == VOID:
                continue
            raise KeyError("In the image with ID {} segment with ID {} is presented in PNG and not presented in JSON."
                           .format(gt_ann["image_id"], label))
        pred_segms[label]["area"] = int(label_cnt)
        pred_labels_set.remove(label)
        if pred_segms[label]["category_id"] not in categories:
            raise KeyError("In the image with ID {} segment with ID {} has unknown category_id {}.".format(
                gt_ann["image_id"], label, pred_segms[label]["category_id"]))
    if len(pred_labels_set) != 0:
        raise KeyError("In the image with ID {} the following segment IDs {} are presented in JSON and not presented "
                       "in PNG.".format(gt_ann["image_id"], list(pred_labels_set)))
    pan_gt_pred = pan_gt.astype(np.uint64) * OFFSET + pan_pred.astype(np.uint64)
    gt_pred_map = {}
    labels, labels_cnt = np.unique(pan_gt_pred, return_counts=True)
    for label, intersection in zip(labels, labels_cnt):
        gt_pred_map[(int(label // OFFSET), int(label % OFFSET))] = int(intersection)
    gt_matched, pred_matched = set(), set()
    for (gt_label, pred_label), intersection in gt_pred_map.items():
        if gt_label not in gt_segms or pred_label not in pred_segms:
            continue
        if gt_segms[gt_label]["iscrowd"] == 1:
            continue
        if gt_segms[gt_label]["category_id"] != pred_segms[pred_label]["category_id"]:
            continue
        union = (pred_segms[pred_label]["area"] + gt_segms[gt_label]["area"] - intersection
                 - gt_pred_map.get((VOID, pred_label), 0))
        iou = intersection / union
        if iou > 0.5:
            stat[gt_segms[gt_label]["category_id"]].tp += 1
            stat[gt_segms[gt_label]["category_id"]].iou += iou
            gt_matched.add(gt_label)
            pred_matched.add(pred_label)
    crowd_labels_dict = {}
    for gt_label, gt_info in gt_segms.items():
        if gt_label in gt_matched:
            continue
        if gt_info["iscrowd"] == 1:
            crowd_labels_dict[gt_info["category_id"]] = gt_label
            continue
        stat[gt_info["category_id"]].fn += 1
    for pred_label, pred_info in pred_segms.items():
        if pred_label in pred_matched:
            continue
        intersection = gt_pred_map.get((VOID, pred_label), 0)
        if pred_info["category_id"] in crowd_labels_dict:
            intersection += gt_pred_map.get((crowd_labels_dict[pred_info["category_id"]], pred_label), 0)
        if intersection / pred_info["area"] > 0.5:
            continue
        stat[pred_info["category_id"]].fp += 1


def pq_average(stat, categories, isthing):
    pq, sq, rq, n = 0, 0, 0, 0
    per_class = {}
    for label, info in categories.items():
        if isthing is not None and isthing != (info["isthing"] == 1):
            continue
        s = stat[label]
        if s.tp + s.fp + s.fn == 0:
            per_class[label] = {"pq": 0.0, "sq": 0.0, "rq": 0.0}
            continue
        n += 1
        pq_class = s.iou / (s.tp + 0.5 * s.fp + 0.5 * s.fn)
        sq_class = s.iou / s.tp if s.tp != 0 else 0
        rq_class = s.tp / (s.tp + 0.5 * s.fp + 0.5 * s.fn)
        per_class[label] = {"pq": pq_class, "sq": sq_class, "rq": rq_class}
        pq, sq, rq = pq + pq_class, sq + sq_class, rq + rq_class
    return {"pq": pq / n, "sq": sq / n, "rq": rq / n, "n": n}, per_class


def pq_stats(gt_json, pred_json, gt_maps, pred_maps):
    """gt_json / pred_json dicts; gt_maps / pred_maps: image id -> raw id map.  Returns the per-category stats."""
    categories = {el["id"]: el for el in gt_json["categories"]}
    pred_annotations = {el["image_id"]: el for el in pred_json["annotations"]}
    for gt_ann in gt_json["annotations"]:
        if gt_ann["image_id"] not in pred_annotations:
            raise Exception("no prediction for the image with id: {}".format(gt_ann["image_id"]))
    stat = defaultdict(PQStatCat)
    for gt_ann in gt_json["annotations"]:
        i = gt_ann["image_id"]
        score_image(stat, gt_ann, gt_maps[i], pred_annotations[i], pred_maps[i], categories)
    return stat


def pq_compute(gt_json, pred_json, gt_maps, pred_maps):
    """panopticapi's result dict and the per-category stats."""
    stat = pq_stats(gt_json, pred_json, gt_maps, pred_maps)
    categories = {el["id"]: el for el in gt_json["categories"]}
    results = {}
    for name, isthing in (("All", None), ("Things", True), ("Stuff", False)):
        results[name], per_class = pq_average(stat, categories, isthing)
        if name == "All":
            results["per_class"] = per_class
    return results, stat
