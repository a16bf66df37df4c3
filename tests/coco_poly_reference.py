"""Plain-Python restatement of pycocotools 2.0's polygon masks, written from its definition: `rleFrPoly` (scale 5,
C truncation toward zero, the 0 / 0 slope of a zero-length edge truncating to INT_MIN as x86-64's cvttsd2si does),
`rleFrBbox`, `frPyObjects`' dispatch and `merge`'s union.  Every float operation is a separately rounded IEEE double
operation, as in pycocotools' x86-64 build.  `contract=True` instead evaluates ys + s * t (and xs + s * t) as one
fused multiply-add, which is what a compiler that contracts would compute; the tests use it to find edges where the
two differ."""
import math
from fractions import Fraction

import numpy as np

SCALE = 5.0
INT_MIN = -2 ** 31


def c_int(q):
    """(int)q on x86-64: truncation toward zero, INT_MIN for NaN and out-of-range values."""
    if q != q or not (-2.0 ** 31 - 1 < q < 2.0 ** 31):
        return INT_MIN
    return int(q)


def grid(c):
    return c_int(SCALE * c + .5)


def _line(base, s, t, contract):
    if contract and s == s:
        return c_int(float(Fraction(base) + Fraction(s) * t) + .5)
    return c_int(base + s * t + .5)


def boundary(xy, contract=False):
    """The boundary points (u, v) of rleFrPoly for one part."""
    k = len(xy) // 2
    x = [grid(float(xy[2 * j])) for j in range(k)]
    y = [grid(float(xy[2 * j + 1])) for j in range(k)]
    if k == 0:
        return [], []
    x.append(x[0])
    y.append(y[0])
    u, v = [], []
    for j in range(k):
        xs, xe, ys, ye = x[j], x[j + 1], y[j], y[j + 1]
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe, ys, ye = xe, xs, ye, ys
        if dx >= dy:
            s = (ye - ys) / dx if dx else float("nan")
            for d in range(dx + 1):
                t = dx - d if flip else d
                u.append(t + xs)
                v.append(_line(ys, s, t, contract))
        else:
            s = (xe - xs) / dy
            for d in range(dy + 1):
                t = dy - d if flip else d
                v.append(t + ys)
                u.append(_line(xs, s, t, contract))
    return u, v


def fr_poly(xy, h, w, contract=False):
    """rleFrPoly: the RLE counts of one polygon part."""
    u, v = boundary(xy, contract)
    a = []
    for j in range(1, len(u)):
        if u[j] == u[j - 1]:
            continue
        xd = float(u[j] if u[j] < u[j - 1] else u[j] - 1)
        xd = (xd + .5) / SCALE - .5
        if math.floor(xd) != xd or xd < 0 or xd > w - 1:
            continue
        yd = float(v[j] if v[j] < v[j - 1] else v[j - 1])
        yd = (yd + .5) / SCALE - .5
        if yd < 0:
            yd = 0
        elif yd > h:
            yd = h
        yd = math.ceil(yd)
        a.append(int(xd) * h + int(yd))
    a.append(h * w)
    a.sort()
    p = 0
    for j in range(len(a)):
        t = a[j]
        a[j] -= p
        p = t
    b = [a[0]]
    j = 1
    while j < len(a):
        if a[j] > 0:
            b.append(a[j])
            j += 1
        else:
            j += 1
            if j < len(a):
                b[-1] += a[j]
                j += 1
    return b


def fr_bbox(bb, h, w, contract=False):
    xs, ys = float(bb[0]), float(bb[1])
    xe, ye = xs + float(bb[2]), ys + float(bb[3])
    return fr_poly([xs, ys, xs, ye, xe, ye, xe, ys], h, w, contract)


def fr_py_objects(seg, h, w, contract=False):
    """frPyObjects of a list segmentation: one RLE counts list per part."""
    if not isinstance(seg, list) or len(seg) == 0 or len(seg[0]) < 4:
        raise ValueError("input type is not supported.")
    if len(seg[0]) == 4:
        return [fr_bbox(p, h, w, contract) for p in seg]
    return [fr_poly(p, h, w, contract) for p in seg]


def decode(counts, h, w):
    """uint8 [h, w] of RLE counts (column-major)."""
    flat = np.zeros(h * w, np.uint8)
    pos = 0
    for i, c in enumerate(counts):
        if i % 2:
            flat[pos:pos + c] = 1
        pos += c
    return flat.reshape(w, h).T.copy()


def encode(mask):
    """RLE counts (zero run first) of a uint8 [h, w] mask."""
    h, w = mask.shape
    counts, pos = [], 0
    for st, ln in runs_of(mask).tolist():
        counts += [st - pos, ln]
        pos = st + ln
    return counts + [h * w - pos]


def runs_of(mask):
    """int64 [n, 2] column-major (start, length) of the runs of ones of a uint8 [h, w] mask."""
    flat = np.asarray(mask, np.uint8).T.reshape(-1).astype(np.int8)
    d = np.diff(np.concatenate(([0], flat, [0])))
    starts, ends = np.flatnonzero(d == 1), np.flatnonzero(d == -1)
    return np.stack((starts, ends - starts), 1).astype(np.int64)


def ann_mask(seg, h, w, contract=False):
    """COCO.annToRLE + decode of a list segmentation: the union of its parts, uint8 [h, w]."""
    m = np.zeros((h, w), np.uint8)
    for c in fr_py_objects(seg, h, w, contract):
        m |= decode(c, h, w)
    return m


def ann_runs(seg, h, w, contract=False):
    return runs_of(ann_mask(seg, h, w, contract))
