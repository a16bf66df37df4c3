"""Seeded synthetic tracking scenes for the MOT evaluation tests and tools/mot_eval_bench.py.

`scene(seed, ...)` returns `(results, frames)`: the tracker's `{track_id: {frame: {"bbox", "score"}}}` and the
loader's frames `[{"gt": {gt_id: x1, y1, x2, y2}}]`.  Ground-truth boxes move at constant velocity and leave for a
while (gaps); hypotheses are the GT boxes with continuous jitter (so no two assignments tie), dropped now and then
(some people most of the time), with track ids that swap between objects or restart, jittered near-duplicates and
false positives.  The frame's `gt` dict lists its objects in a shuffled order.
"""
import numpy as np


def scene(seed, n_frames=40, n_objects=10, width=1920.0, height=1080.0, size=(60.0, 150.0), jitter=0.06,
          p_drop=0.08, p_swap=0.01, p_restart=0.01, p_dup=0.05, fp_rate=0.5, p_gap=0.01, gt_box=np.asarray):
    rng = np.random.default_rng(seed)
    n = n_objects
    wh = np.stack([rng.uniform(0.5, 1.5, n) * size[0], rng.uniform(0.5, 1.5, n) * size[1]], 1)
    pos = np.stack([rng.uniform(0, width, n), rng.uniform(0, height, n)], 1)
    vel = rng.normal(0, 3, (n, 2))
    gt_id = np.arange(n) + 1
    next_gt = n + 1
    track = np.arange(n)
    next_track = n
    results = {}
    frames = []
    absent = np.zeros(n, dtype=np.int64)
    drop = rng.choice([p_drop, 0.5, 0.9], n, p=[0.7, 0.15, 0.15])     # some people are mostly missed
    for f in range(n_frames):
        pos += vel
        out = (pos[:, 0] < -wh[:, 0]) | (pos[:, 0] > width) | (pos[:, 1] < -wh[:, 1]) | (pos[:, 1] > height)
        for i in np.nonzero(out)[0]:                      # a new person enters
            pos[i] = rng.uniform(0, width), rng.uniform(0, height)
            gt_id[i], next_gt = next_gt, next_gt + 1
            track[i], next_track = next_track, next_track + 1
        absent = np.maximum(absent - 1, 0)
        absent[rng.random(n) < p_gap] = rng.integers(1, 6)
        for i in np.nonzero(rng.random(n) < p_swap)[0]:
            j = rng.integers(n)
            track[i], track[j] = track[j], track[i]
        for i in np.nonzero(rng.random(n) < p_restart)[0]:
            track[i], next_track = next_track, next_track + 1
        boxes = np.concatenate([pos, pos + wh], 1).astype(np.float32)
        gt = {}
        for i in rng.permutation(n):
            if not absent[i]:
                gt[int(gt_id[i])] = gt_box(boxes[i])
        frames.append({"gt": gt})

        def emit(t, box):
            results.setdefault(int(t), {})[f] = {"bbox": np.asarray(box, np.float32), "score": np.float32(1.0)}

        for i in range(n):
            if absent[i] or rng.random() < drop[i]:
                continue
            emit(track[i], boxes[i] + rng.normal(0, jitter, 4) * np.r_[wh[i], wh[i]])
            if rng.random() < p_dup:
                emit(next_track, boxes[i] + rng.normal(0, 2 * jitter, 4) * np.r_[wh[i], wh[i]])
                next_track += 1
        for _ in range(rng.poisson(fp_rate)):
            x, y = rng.uniform(0, width), rng.uniform(0, height)
            emit(next_track, np.r_[x, y, x + size[0], y + size[1]])
            next_track += 1
    return results, frames


def clumps(seed, n_frames=12, n_clumps=150, per=(2, 6), jitter=4.0, p_drop=0.1, p_restart=0.3, fp_rate=2.0, cols=15):
    """Crowded frames: `n_clumps` groups of 2-6 people standing almost on top of each other (every pair inside a
    group valid, none across groups), about 600 objects per frame with the defaults.  Track ids restart often, so most
    frames have residual assignment problems of several boxes on each side."""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(per[0], per[1] + 1, n_clumps)
    clump = np.repeat(np.arange(n_clumps), sizes)
    n = len(clump)
    base = np.stack([(clump % cols) * 250.0, (clump // cols) * 400.0], 1)
    vel = np.repeat(rng.normal(0, 2, (n_clumps, 2)), sizes, axis=0)
    track = np.arange(n)
    next_track = n
    results, frames = {}, []
    for f in range(n_frames):
        base += vel
        boxes = (np.concatenate([base, base + [100.0, 200.0]], 1) + rng.normal(0, jitter, (n, 4))).astype(np.float32)
        frames.append({"gt": {int(i) + 1: boxes[i] for i in rng.permutation(n)}})
        for i in np.nonzero(rng.random(n) < p_restart)[0]:
            track[i], next_track = next_track, next_track + 1
        for i in range(n):
            if rng.random() >= p_drop:
                box = boxes[i] + rng.normal(0, jitter, 4)
                results.setdefault(int(track[i]), {})[f] = {"bbox": box.astype(np.float32)}
        for _ in range(rng.poisson(fp_rate)):
            x, y = rng.uniform(0, cols * 250.0), rng.uniform(0, 4000.0)
            results[next_track] = {f: {"bbox": np.asarray([x, y, x + 100, y + 200], np.float32)}}
            next_track += 1
    return results, frames
