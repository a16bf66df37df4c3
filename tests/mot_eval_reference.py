"""Event-level restatement of the MOTChallenge metrics that motmetrics 1.2.0 computes for the reference's
get_mot_accum / evaluate_mot_accums (src/trackformer/util/track_utils.py:354-417), in Python dicts, numpy and scipy.

The oracle of tests/test_mot_eval_*.py; product code never imports it.  The rules:

- distances: boxes x1, y1, x2, y2 -> x, y, w, h in float32 (w = fl32(x2 - x1)), promoted to float64; IoU of the
  extents [x, x + w] (motmetrics.distances.iou_matrix); d = 1 - IoU, valid iff d <= 0.5.
- per frame (MOTAccumulator.update): re-establish each object's previous partner when it is present, unmasked and
  valid, objects in the frame's order; then the assignment of the remaining valid pairs through motmetrics'
  add_expensive_edges (invalid pairs cost 2 r (max |valid d| + 1) + 1, r = min(rows, cols)) and
  scipy.optimize.linear_sum_assignment; SWITCH when the object had a different previous partner; MISS / FP for the
  rest.
- counts and ratios as motmetrics.metrics.motchallenge_metrics; IDTP is the maximum-weight matching of tp(o, h), the
  number of frames in which (o, h) is a valid pair.
"""
import numpy as np
from scipy.optimize import linear_sum_assignment

MAX_IOU = 0.5


def to_xywh(boxes):
    b = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    return np.stack((b[:, 0], b[:, 1], b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]), axis=1)


def iou_distance(objs, hyps, max_iou=MAX_IOU):
    """[n_obj, n_hyp] float64 d, NaN where invalid (motmetrics.distances.iou_matrix)."""
    a = np.asarray(objs, np.float64).reshape(-1, 4)[:, None]
    b = np.asarray(hyps, np.float64).reshape(-1, 4)[None, :]
    a_min, a_max = a[..., :2], a[..., :2] + a[..., 2:]
    b_min, b_max = b[..., :2], b[..., :2] + b[..., 2:]
    i_size = np.maximum(np.minimum(a_max, b_max) - np.maximum(a_min, b_min), 0)
    i_vol = i_size[..., 0] * i_size[..., 1]
    a_size, b_size = np.maximum(a_max - a_min, 0), np.maximum(b_max - b_min, 0)
    u_vol = a_size[..., 0] * a_size[..., 1] + b_size[..., 0] * b_size[..., 1] - i_vol
    with np.errstate(divide="ignore", invalid="ignore"):
        iou = np.where(i_vol == 0, 0.0, i_vol / u_vol)
    d = 1.0 - iou
    return np.where(d > max_iou, np.nan, d)


def expensive_edges(costs):
    valid = np.isfinite(costs)
    if valid.all():
        return costs.copy()
    if not valid.any():
        return np.zeros_like(costs)
    r = min(costs.shape)
    big = 2 * r * (np.max(np.abs(costs[valid])) + 1) + 1
    return np.where(valid, costs, big)


class Accumulator:
    """MOTAccumulator without the extended event types: events are (frame, type, oid, hid, d)."""

    def __init__(self):
        self.m = {}
        self.events = []
        self.frame = 0
        self.n_hyp = 0
        self.tp = {}

    def update(self, oids, hids, dists):
        oids, hids = list(oids), list(hids)
        d = np.asarray(dists, np.float64).reshape(len(oids), len(hids)).copy()
        f = self.frame
        self.frame += 1
        self.n_hyp += len(hids)
        for i, j in zip(*np.nonzero(np.isfinite(d))):
            self.tp[(oids[i], hids[j])] = self.tp.get((oids[i], hids[j]), 0) + 1
        omask, hmask = [False] * len(oids), [False] * len(hids)
        if oids and hids:
            for i, o in enumerate(oids):
                if o not in self.m:
                    continue
                js = [j for j, h in enumerate(hids) if h == self.m[o] and not hmask[j]]
                if js and np.isfinite(d[i, js[0]]):
                    omask[i] = hmask[js[0]] = True
                    self.events.append((f, "MATCH", o, hids[js[0]], d[i, js[0]]))
            d[np.asarray(omask), :] = np.nan
            d[:, np.asarray(hmask)] = np.nan
            for i, j in zip(*linear_sum_assignment(expensive_edges(d))):
                if not np.isfinite(d[i, j]):
                    continue
                o, h = oids[i], hids[j]
                kind = "SWITCH" if o in self.m and self.m[o] != h else "MATCH"
                self.events.append((f, kind, o, h, d[i, j]))
                self.m[o] = h
                omask[i] = hmask[j] = True
        for i, o in enumerate(oids):
            if not omask[i]:
                self.events.append((f, "MISS", o, None, np.nan))
        for j, h in enumerate(hids):
            if not hmask[j]:
                self.events.append((f, "FP", None, h, np.nan))


def accumulate(results, frames_gt):
    """get_mot_accum: frames_gt[f] is frame f's {gt_id: x1, y1, x2, y2 box}; results {track_id: {frame: {"bbox"}}}."""
    acc = Accumulator()
    for f, gt in enumerate(frames_gt):
        oids = list(gt.keys())
        objs = to_xywh([np.asarray(gt[o], np.float32).reshape(-1)[:4] for o in oids]) if oids else np.zeros((0, 4))
        hids = [t for t, track in results.items() if f in track]
        hyps = (to_xywh([np.asarray(results[t][f]["bbox"], np.float32)[:4] for t in hids]) if hids
                else np.zeros((0, 4)))
        acc.update(oids, hids, iou_distance(objs, hyps))
    return acc


def counts(acc):
    ev = acc.events
    kinds = [e[1] for e in ev]
    out = {k: kinds.count(t) for k, t in (("matches", "MATCH"), ("switches", "SWITCH"), ("misses", "MISS"),
                                          ("fp", "FP"))}
    out["sum_d"] = float(sum(e[4] for e in ev if e[1] in ("MATCH", "SWITCH")))
    out["num_objects"] = out["matches"] + out["switches"] + out["misses"]
    out["num_predictions"] = acc.n_hyp
    per_obj = {}
    for e in ev:
        if e[2] is not None:
            per_obj.setdefault(e[2], []).append(e[1] != "MISS")
    out["gt"] = len(per_obj)
    mt = pt = ml = fm = 0
    for hits in per_obj.values():
        ratio = sum(hits) / len(hits)
        if ratio >= 0.8:
            mt += 1
        elif ratio < 0.2:
            ml += 1
        else:
            pt += 1
        idx = [i for i, h in enumerate(hits) if h]
        if idx:
            span = hits[idx[0]:idx[-1] + 1]
            fm += sum(1 for a, b in zip(span, span[1:]) if a and not b)
    out.update(mt=mt, pt=pt, ml=ml, fm=fm)
    oids = sorted({o for o, _ in acc.tp}, key=repr)
    hids = sorted({h for _, h in acc.tp}, key=repr)
    w = np.zeros((len(oids), len(hids)))
    oi, hi = {o: i for i, o in enumerate(oids)}, {h: j for j, h in enumerate(hids)}
    for (o, h), n in acc.tp.items():
        w[oi[o], hi[h]] = n
    r, c = linear_sum_assignment(-w) if w.size else ([], [])
    out["idtp"] = int(w[r, c].sum()) if w.size else 0
    return out


def metrics(c):
    """motmetrics' motchallenge_metrics from counts (division by zero as numpy gives it)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        n_obj, n_pred = np.float64(c["num_objects"]), np.float64(c["num_predictions"])
        det = np.float64(c["matches"] + c["switches"])
        idtp = np.float64(c["idtp"])
        return {
            "idf1": 2 * idtp / (n_obj + n_pred), "idp": idtp / n_pred, "idr": idtp / n_obj,
            "recall": det / n_obj, "precision": det / (det + c["fp"]),
            "num_unique_objects": c["gt"], "mostly_tracked": c["mt"], "partially_tracked": c["pt"],
            "mostly_lost": c["ml"], "num_false_positives": c["fp"], "num_misses": c["misses"],
            "num_switches": c["switches"], "num_fragmentations": c["fm"],
            "mota": 1.0 - (c["misses"] + c["switches"] + c["fp"]) / n_obj, "motp": c["sum_d"] / det,
        }


def evaluate(named):
    """{name: counts} -> {name: metrics} plus OVERALL (counts summed, ratios recomputed)."""
    out = {n: metrics(c) for n, c in named.items()}
    total = {k: sum(c[k] for c in named.values()) for k in next(iter(named.values()))}
    out["OVERALL"] = metrics(total)
    return out
