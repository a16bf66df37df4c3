#!/usr/bin/env python
"""Frame-ingest fixtures recorded FROM THE REFERENCE (build container only).

Runs seeded synthetic uint8 images (noise, smooth ramps, hard 0 / 255 edges) through the reference's own validation
transform -- `Compose(make_coco_transforms('val', img_transform))` followed by its `normalize`
(src/trackformer/datasets/coco.py:270-312, the very objects datasets/tracking/mot17_sequence.py:48,71 applies per frame)
-- and stores, per case, the input bytes, the resized bytes, the normalised float image and both sizes in
tests/golden/frame_ingest.npz.  Small `img_transform` settings keep the file small; the cases cover landscape and
portrait reduction, enlargement, the max_size cap, a frame already at the target short side, and odd sizes.

`pycocotools` is not importable here and the transform does not use it: it is stubbed like `visdom`.
"""
import os
import sys
import types
from argparse import Namespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

# name: (H, W, val_width, max_size)
CASES = {
    "landscape_down": (108, 192, 60, 100),         # 16:9: the cap takes effect
    "portrait_down": (192, 108, 60, 100),          # the same shape upright
    "up_4x3": (30, 40, 60, 100),                   # enlargement, no cap -> 60x80
    "up_portrait_cap": (32, 20, 60, 90),           # enlargement, capped: round (short side) and truncation (long side)
    "already_at_target": (60, 91, 60, 100),        # short side is the target: returned unchanged, look-up only
    "wide_cap": (60, 150, 60, 100),                # short side at the target, but the cap shrinks both axes
    "odd_sizes": (61, 109, 50, 83),
    "strong_reduction": (201, 259, 20, 33),        # scale ~ 10: ksize 23
    "tiny": (7, 5, 9, 100),
}


def synthetic(h, w, seed):
    """uint8 [h, w, 3]: top third hard 0 / 255 blocks, middle third smooth ramps, the rest noise"""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    a, b = h // 3, 2 * h // 3
    img[:a] = np.where(rng.random((a, w, 1)) > 0.5, 255, 0)
    yy, xx = np.mgrid[a:b, 0:w]
    for c in range(3):
        img[a:b, :, c] = ((xx * (c + 1) * 255 // max(w - 1, 1) + yy * 3) % 256).astype(np.uint8)
    return img


def main():
    from make_golden_model import import_reference
    for name in ("pycocotools", "pycocotools.coco", "pycocotools.mask", "pycocotools.cocoeval"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["pycocotools.coco"].COCO = type("COCO", (), {})
    sys.modules["pycocotools.cocoeval"].COCOeval = type("COCOeval", (), {})
    sys.modules["pycocotools"].mask = sys.modules["pycocotools.mask"]
    import_reference()
    from PIL import Image
    from trackformer.datasets.coco import make_coco_transforms
    from trackformer.datasets.transforms import Compose

    out = {"names": np.asarray(list(CASES))}
    for seed, (name, (h, w, val_width, max_size)) in enumerate(CASES.items()):
        pair = make_coco_transforms("val", Namespace(val_width=val_width, max_size=max_size), overflow_boxes=True)
        frame = synthetic(h, w, seed)
        img, _ = Compose(pair)(Image.fromarray(frame))           # the datasets' self.transforms: (resize, normalize)
        resized, _ = pair[0](Image.fromarray(frame))             # its first half alone, for the bytes in between
        rw, rh = resized.size
        assert tuple(img.shape) == (3, rh, rw)
        out[f"{name}_frame"] = frame
        out[f"{name}_resized"] = np.asarray(resized)
        out[f"{name}_img"] = img.numpy()
        out[f"{name}_settings"] = np.asarray([val_width, max_size], np.int64)
        out[f"{name}_size"] = np.asarray([rh, rw], np.int64)
        out[f"{name}_orig_size"] = np.asarray([h, w], np.int64)
        print(f"{name}: {h}x{w} -> {rh}x{rw}")
    path = os.path.join(HERE, "frame_ingest.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
