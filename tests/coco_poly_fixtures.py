"""Seeded polygon segmentations for the polygon-mask tests (numpy only): convex, non-convex, self-intersecting,
repeated and collinear vertices, vertices outside the image on every side (negative fractional coordinates
included), 2-point and odd-length parts, overlapping multi-part annotations, box lists, vertices on x = w - 1 and
y = h, and edges on which a contracted ys + s * t + .5 gives another mask (grid values found by an exact search)."""
import numpy as np

# (xs, ys, xe, ye) on pycocotools' 5x grid of a 1080 x 1920 image: edges whose mask differs when ys + s * t is one
# fused multiply-add, found by tests/test_coco_poly_cpu.py's fma_sensitive_edges search (seed 7)
FMA_EDGES = [(1005, 2613, 9269, 39), (953, 5235, 8273, 285), (2626, 3592, 9360, 1113), (3568, 4985, 9112, 332),
             (2551, 3758, 9279, 1306), (1935, 4693, 9487, 1141)]


def from_grid(g):
    """A coordinate c with (int)(5 c + .5) == g (truncation toward zero)."""
    return g / 5.0 if g >= 0 else (g - 1.0) / 5.0


def fma_polygons():
    """A triangle on each FMA-sensitive edge (1080 x 1920)."""
    out = []
    for xs, ys, xe, ye in FMA_EDGES:
        c = [from_grid(v) for v in (xs, ys, xe, ye)]
        out.append([[c[0], c[1], c[2], c[3], c[0], c[3]]])
    return out


def _part(rng, h, w, kind):
    n = int(rng.integers(3, 12)) if kind != "long" else int(rng.integers(8, 81))
    cx, cy = rng.uniform(-0.1 * w, 1.1 * w), rng.uniform(-0.1 * h, 1.1 * h)
    r = rng.uniform(2, max(3.0, 0.5 * min(h, w)))
    if kind == "convex":
        ang = np.sort(rng.uniform(0, 2 * np.pi, n))
        pts = np.stack((cx + r * np.cos(ang), cy + r * np.sin(ang)), 1)
    elif kind in ("star", "long"):
        ang = np.sort(rng.uniform(0, 2 * np.pi, n))
        rad = r * rng.uniform(0.2, 1.0, n)
        pts = np.stack((cx + rad * np.cos(ang), cy + rad * np.sin(ang)), 1)
    elif kind == "random":                                    # self-intersecting
        pts = np.stack((rng.uniform(-0.2 * w, 1.2 * w, n), rng.uniform(-0.2 * h, 1.2 * h, n)), 1)
    elif kind == "outside":                                   # beyond every side, negative fractional values
        pts = np.stack((rng.uniform(-3.7, 2.2, n) * w - rng.uniform(0, 1, n),
                        rng.uniform(-2.3, 3.1, n) * h - rng.uniform(0, 1, n)), 1)
    elif kind == "edge":                                      # vertices on x = w - 1 and y = h, and on 0
        xs = rng.choice([0.0, w - 1.0, w - 1.0, w, rng.uniform(0, w)], n)
        ys = rng.choice([0.0, float(h), float(h), h - 1.0, rng.uniform(0, h)], n)
        pts = np.stack((xs, ys), 1)
    elif kind == "integer":
        pts = np.stack((rng.integers(-2, w + 2, n), rng.integers(-2, h + 2, n)), 1).astype(np.float64)
    else:
        raise ValueError(kind)
    if rng.random() < 0.3:                                    # repeated vertices
        i = int(rng.integers(0, n))
        pts = np.insert(pts, i, pts[i], 0)
    if rng.random() < 0.3:                                    # a collinear vertex
        i = int(rng.integers(0, len(pts) - 1))
        pts = np.insert(pts, i + 1, (pts[i] + pts[i + 1]) / 2, 0)
    if rng.random() < 0.5:
        pts = np.round(pts, int(rng.integers(0, 3)))
    return [float(v) for v in pts.reshape(-1)]


KINDS = ("convex", "star", "random", "outside", "edge", "integer", "long")


def segmentation(rng, h, w):
    """One list segmentation: 1 - 4 polygon parts (later parts may be 2-point or odd-length), or a box list."""
    if rng.random() < 0.12:
        nb = int(rng.integers(1, 4))
        return [[float(np.round(rng.uniform(-0.2 * w, w), 2)), float(np.round(rng.uniform(-0.2 * h, h), 2)),
                 float(np.round(rng.uniform(0, 0.6 * w), 2)), float(np.round(rng.uniform(0, 0.6 * h), 2))]
                for _ in range(nb)]
    parts = [_part(rng, h, w, KINDS[int(rng.integers(0, len(KINDS)))]) for _ in range(int(rng.integers(1, 5)))]
    for i in range(1, len(parts)):
        u = rng.random()
        if u < 0.1:
            parts[i] = parts[i][:4]                           # a 2-point polygon
        elif u < 0.2:
            parts[i] = parts[i] + [float(rng.uniform(0, w))]  # odd length: the last number is ignored
    return parts


def segmentations(seed, n, h, w):
    rng = np.random.default_rng(seed)
    return [segmentation(rng, h, w) for _ in range(n)]


def coco_val_like(seed, n_images=5000, per_image=7.2):
    """A COCO-val-sized ground truth with polygon masks: n_images images of COCO-like sizes and about per_image
    annotations each, 1 - 4 parts of 8 - 80 vertices around an object-sized centre (seeded)."""
    rng = np.random.default_rng(seed)
    images, anns = [], []
    sizes = [(480, 640), (640, 480), (427, 640), (640, 427), (375, 500), (500, 375), (612, 612)]
    for i in range(n_images):
        h, w = sizes[int(rng.integers(0, len(sizes)))]
        images.append({"id": i + 1, "height": h, "width": w})
        for _ in range(int(rng.poisson(per_image))):
            cx, cy = rng.uniform(0, w), rng.uniform(0, h)
            r = float(np.exp(rng.uniform(np.log(4), np.log(0.45 * min(h, w)))))
            parts = []
            for _ in range(int(rng.integers(1, 5))):
                n = int(rng.integers(8, 81))
                ang = np.sort(rng.uniform(0, 2 * np.pi, n))
                rad = r * rng.uniform(0.5, 1.0, n)
                px, py = cx + rng.normal(0, r / 2), cy + rng.normal(0, r / 2)
                pts = np.stack((np.clip(px + rad * np.cos(ang), 0, w), np.clip(py + rad * np.sin(ang), 0, h)), 1)
                parts.append([float(v) for v in np.round(pts, 2).reshape(-1)])
            anns.append({"id": len(anns) + 1, "image_id": i + 1, "category_id": int(rng.integers(1, 4)),
                         "iscrowd": 0, "area": float(np.pi * r * r), "bbox": [cx - r, cy - r, 2 * r, 2 * r],
                         "segmentation": parts})
    return {"images": images, "annotations": anns,
            "categories": [{"id": c, "name": str(c)} for c in (1, 2, 3)]}
