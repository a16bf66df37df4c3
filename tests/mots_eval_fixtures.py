"""Seeded synthetic MOTS sequences for the MOTS evaluation tests and tools/mots_eval_bench.py: GT masks in the
`mots.load_results` form (class 2 objects, class 10 ignore regions) and tracker-style results, every mask a COCO RLE
made straight from its foreground intervals (no dense masks).

Each object owns a vertical slot of the image, so masks of one side never overlap.  `style="person"`: one row range per
column; `style="fragmented"`: many short runs per column, like masks of random weights.  Hypotheses copy the GT with
jitter (sometimes far enough to fall under IoU 0.5), misses, id switches, false positives in free slots, and
hypotheses in the ignore slot that lie partly inside the frame's ignore region."""
import numpy as np

from trackformer_b200 import mots


def rle(iv, h, w):
    """COCO RLE of sorted, disjoint column-major intervals iv [n, 2] (abutting ones merged as pycocotools would)"""
    n = h * w
    iv = np.asarray(iv, np.int64).reshape(-1, 2)
    if len(iv):
        keep = np.ones(len(iv), bool)
        keep[1:] = iv[1:, 0] != iv[:-1, 1]
        starts = iv[keep, 0]
        ends = iv[np.append(keep[1:], True), 1]                # the last end of each merged group
        edges = np.concatenate(([0], np.stack([starts, ends], 1).reshape(-1), [n]))
        cnts = np.diff(edges)
        if cnts[-1] == 0:
            cnts = cnts[:-1]
    else:
        cnts = np.asarray([n], np.int64)
    return {"size": [h, w], "counts": mots._string(cnts.astype(np.int64))}


def _column_runs(cols, y0, y1, h, rng, fragmented):
    """intervals of rows [y0, y1) in each column (fragmented: short runs with gaps >= 3)"""
    out = []
    for c in cols:
        if fragmented:
            edges = np.sort(rng.choice(np.arange(y0, y1, 4), size=2 * max(1, (y1 - y0) // 16), replace=False))
            rows = edges.reshape(-1, 2)
            rows[:, 1] = np.maximum(rows[:, 1] - 1, rows[:, 0] + 1)
        else:
            rows = np.asarray([[y0, y1]])
        out.append(rows + c * h)
    return np.concatenate(out) if out else np.zeros((0, 2), np.int64)


def _jitter(iv, h, rng, amount, whole):
    """move every run end by up to `amount` rows (whole: the whole mask by one amount), clipped to its column; drop
    empty runs.  Runs stay disjoint: per-end moves are smaller than half the gaps, a whole move keeps the order."""
    if not len(iv):
        return iv
    col = iv[:, 0] // h
    sh = rng.integers(-amount, amount + 1, size=(1, 1) if whole else iv.shape)
    out = np.clip(iv + sh, col[:, None] * h, col[:, None] * h + h)
    return out[out[:, 1] > out[:, 0]]


def scene(seed, n_frames=20, n_objects=6, size=(96, 160), style="person", p_miss=0.1, p_fp=0.3, p_switch=0.03,
          p_ignore=0.5, p_far=0.1, as_rle=True, chain=None):
    """(results, gt): results {track: {frame: {"mask"}}}, gt {id: {frame: {"mask", "class_id"}}} (load_results form).
    chain=(life_lo, life_hi, gap_lo, gap_hi): each of the n_objects slots holds a succession of objects, each alive for
    a uniform number of frames in [life_lo, life_hi) after a gap in [gap_lo, gap_hi); without it, object k alone
    holds slot k for one span."""
    h, w = size
    rng = np.random.default_rng(seed)
    frag = style == "fragmented"
    n_slots = n_objects + 3                               # objects, two free slots for false positives, ignore
    sw = w // n_slots
    assert sw >= 4, "image too narrow for the objects"
    if chain is None:
        first = rng.integers(0, max(1, n_frames // 2), n_objects)
        last = np.minimum(n_frames, first + rng.integers(max(2, n_frames // 3), n_frames + 1, n_objects))
        spans = [[(int(first[k]), int(last[k]), k)] for k in range(n_objects)]
    else:
        spans, n_ids = [], 0
        for _ in range(n_objects):
            at, slot = 0, []
            while True:
                at += int(rng.integers(chain[2], chain[3]))
                if at >= n_frames:
                    break
                end = min(n_frames, at + int(rng.integers(chain[0], chain[1])))
                slot.append((at, end, n_ids))
                n_ids, at = n_ids + 1, end
            spans.append(slot)
    n_ids = sum(len(sp) for sp in spans)
    gt, results = {}, {}
    track_of = list(range(n_ids))
    next_track = n_ids
    ign_slot = n_slots - 1

    def put(d, key, f, iv, extra=None):
        m = rle(iv, h, w) if as_rle else _dense(iv, h, w)
        d.setdefault(key, {})[f] = {"mask": m, **(extra or {})}

    for f in range(n_frames):
        for k in range(n_objects):
            alive = [i for b, e, i in spans[k] if b <= f < e]
            if not alive:
                continue
            obj = alive[0]
            c0 = k * sw + int(rng.integers(0, max(1, sw // 4)))
            c1 = min((k + 1) * sw, c0 + max(2, sw - sw // 4 - int(rng.integers(0, max(1, sw // 4)))))
            y0 = int(rng.integers(0, h // 3))
            y1 = min(h, y0 + h // 2 + int(rng.integers(0, h // 3)))
            iv = _column_runs(range(c0, c1), y0, y1, h, rng, frag)
            put(gt, obj + 1, f, iv, {"class_id": 2})
            if rng.random() < p_switch:
                track_of[obj], next_track = next_track, next_track + 1
            if rng.random() < p_miss:
                continue
            far = rng.random() < p_far
            put(results, track_of[obj], f, _jitter(iv, h, rng, (y1 - y0) // 2 if far else (1 if frag else 3), far))
        for slot in (n_objects, n_objects + 1):
            if rng.random() < p_fp:
                y0 = int(rng.integers(0, h // 2))
                iv = _column_runs(range(slot * sw, slot * sw + sw // 2), y0, y0 + h // 3, h, rng, frag)
                put(results, next_track, f, iv)
                next_track += 1
        if rng.random() < p_ignore:
            y0 = int(rng.integers(0, h // 2))
            put(gt, 10000, f, _column_runs(range(ign_slot * sw, ign_slot * sw + sw), y0, y0 + h // 3, h, rng,
                                           False), {"class_id": 10})
            if rng.random() < 0.7:                            # partly inside the ignore region
                y = int(rng.integers(max(0, y0 - h // 4), y0 + h // 6))
                put(results, next_track, f, _column_runs(range(ign_slot * sw, ign_slot * sw + sw // 2), y,
                                                         min(h, y + h // 4), h, rng, frag))
                next_track += 1
    return results, gt


def _dense(iv, h, w):
    flat = np.zeros(h * w, bool)
    for s, e in np.asarray(iv).reshape(-1, 2):
        flat[s:e] = True
    return flat.reshape(w, h).T.copy()


# MOTS20 train: frames and frame size per sequence
MOTS20_TRAIN = [("MOTS20-02", 600, (1080, 1920)), ("MOTS20-05", 837, (480, 640)), ("MOTS20-09", 525, (1080, 1920)),
                ("MOTS20-11", 900, (1080, 1920))]


def _mots20_sequence(args):
    i, n_frames, size, style = args
    return (*scene(60 + i, n_frames=n_frames, n_objects=11, size=size, style=style, p_switch=0.005,
                   chain=(70, 190, 0, 40)), n_frames)


def mots20_workload(style, pool=None):
    """{name: (results, gt, n_frames)} the size of MOTS20 train (about 26,900 GT masks over about 230 tracks in 2,862
    frames): 11 slots per sequence, each holding a succession of people alive 70-190 frames after gaps of 0-40
    frames, which gives 26,753 GT masks over 226 GT tracks.  `pool`: a multiprocessing pool to build the sequences in
    parallel."""
    args = [(i, f, size, style) for i, (_, f, size) in enumerate(MOTS20_TRAIN)]
    seqs = pool.map(_mots20_sequence, args) if pool is not None else [_mots20_sequence(a) for a in args]
    return {n: v for (n, _, _), v in zip(MOTS20_TRAIN, seqs)}
