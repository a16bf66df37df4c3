"""Dense restatement of the MOTS metrics of trackformer_b200.mots_eval, in numpy: the oracle of
tests/test_mots_eval_*.py; product code never imports it.

Every mask is decoded with `mots.decode` to a dense bool array.  Per frame: IoU of every (GT, hypothesis) pair from
pixel counts (one histogram of the frame's two label maps), candidate iff inter > 0 and 2 inter >= union, d = 1 - inter / union; a hypothesis without a candidate
and with 2 |h & ignore| > |h| is dropped.  The distance matrices go to tests/mot_eval_reference.py's `Accumulator`
(motmetrics 1.2.0's rules), and the MOTS quantities follow from its counts.  The sum of d is taken in one fixed
order, per frame over its objects in order and then over the frames, so it can be compared bit for bit.
"""
import numpy as np

import mot_eval_reference as mer
from trackformer_b200 import mots

GT_CLASS, IGNORE_CLASS = 2, 10


def _dense(m):
    return mots.decode(m) if isinstance(m, dict) else np.asarray(m, bool)


def frame_distances(args):
    """(gt masks, ignore masks, hypothesis masks) of one frame -> (d [n_gt, n_hyp] with NaN off the candidates, kept
    hypothesis indices).  Each mask is decoded to a dense bool array and painted into a label map of its side (GT
    row + 1, ignore regions one label after the GT rows; hypothesis column + 1); one histogram of the label pairs gives
    every intersection, the margins the areas."""
    gt, ignore, hyps = args
    no, nh = len(gt), len(hyps)
    glab = hlab = None
    for side, masks, first in ((0, gt, 1), (0, ignore, no + 1), (1, hyps, 1)):
        for k, m in enumerate(masks):
            px = _dense(m).reshape(-1)
            if side == 0:
                glab = np.zeros(px.size, np.int64) if glab is None else glab
                assert not glab[px].any(), "GT masks overlap"
                glab[px] = first + (k if masks is gt else 0)
            else:
                hlab = np.zeros(px.size, np.int64) if hlab is None else hlab
                assert not hlab[px].any(), "hypothesis masks overlap"
                hlab[px] = first + k
    if nh == 0:
        return np.zeros((no, 0)), []
    if glab is None:
        glab = np.zeros_like(hlab)
    joint = np.bincount(glab * (nh + 1) + hlab, minlength=(no + 2) * (nh + 1)).reshape(no + 2, nh + 1)
    inter = joint[1:no + 1, 1:]
    area_g, area_h = joint[1:no + 1].sum(1), joint[:, 1:].sum(0)
    uni = area_g[:, None] + area_h[None, :] - inter
    cand = (inter > 0) & (2 * inter >= uni)
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.where(cand, 1.0 - inter / np.maximum(uni, 1), np.nan)
    ign = joint[no + 1, 1:]
    keep = [j for j in range(nh) if cand[:, j].any() or not ignore or not 2 * int(ign[j]) > int(area_h[j])]
    return d, keep


def frame_update(acc, oids, hids, d, keep):
    """one frame into the Accumulator; returns the number of removed hypotheses and the frame's sum of d"""
    first = len(acc.events)
    acc.update(oids, [hids[j] for j in keep], d[:, keep])
    dev = {e[2]: e[4] for e in acc.events[first:] if e[1] in ("MATCH", "SWITCH")}
    sum_d = 0.0
    for o in oids:                                       # the frame's sum in object order
        sum_d += dev.get(o, 0.0)
    return len(hids) - len(keep), sum_d


def accumulate(results, gt, num_frames, pool=None):
    """results {track: {frame: {"mask"}}}, gt the mots.load_results form; objects of a frame in the dict's order.
    `pool`: a multiprocessing pool for the frames' dense work (the matching itself runs here, frame by frame)."""
    frames = []
    for f in range(num_frames):
        objs = [(i, fr[f]["mask"]) for i, fr in gt.items() if f in fr and fr[f].get("class_id", GT_CLASS) == GT_CLASS]
        ign = [fr[f]["mask"] for fr in gt.values() if f in fr and fr[f].get("class_id") == IGNORE_CLASS]
        hyps = [(t, tr[f]["mask"]) for t, tr in results.items()
                if f in tr and tr[f].get("class_id", GT_CLASS) == GT_CLASS]
        frames.append((objs, ign, hyps))
    work = [([m for _, m in o], ig, [m for _, m in h]) for o, ig, h in frames]
    dists = pool.imap(frame_distances, work, chunksize=8) if pool is not None else map(frame_distances, work)
    acc = mer.Accumulator()
    removed, sum_d = 0, 0.0
    for (objs, _, hyps), (d, keep) in zip(frames, dists):
        r, s = frame_update(acc, [o for o, _ in objs], [h for h, _ in hyps], d, keep)
        removed, sum_d = removed + r, sum_d + s
    return acc, removed, sum_d


def counts(acc, removed, sum_d):
    """mot_eval_reference's counts, with the removed hypotheses and sum of d in a fixed order: per frame over its
    objects in order, then over the frames"""
    c = mer.counts(acc)
    assert abs(c["sum_d"] - sum_d) <= 1e-9 * max(1.0, sum_d)
    c.update(removed=removed, sum_d=sum_d)
    return c


def metrics(c):
    """the MOTS quantities and mot_eval's ratios from counts"""
    m = mer.metrics(c)
    with np.errstate(divide="ignore", invalid="ignore"):
        tp = np.float64(c["matches"] + c["switches"])
        gt_dets = np.float64(c["num_objects"])
        tp_soft = tp - c["sum_d"]
        m.update(smotsa=(tp_soft - c["fp"] - c["switches"]) / gt_dets, motsa=(tp - c["fp"] - c["switches"]) / gt_dets,
                 motsp=tp_soft / tp, num_detections=c["matches"] + c["switches"], num_ignored=c["removed"])
    return m


def evaluate(named):
    """{name: counts} -> {name: metrics} plus OVERALL (counts summed, ratios recomputed)."""
    out = {n: metrics(c) for n, c in named.items()}
    total = {k: sum(c[k] for c in named.values()) for k in next(iter(named.values()))}
    out["OVERALL"] = metrics(total)
    return out
