#!/usr/bin/env python
"""Panoptic post-processing golden fixtures recorded FROM THE REFERENCE (build container only).

Runs the reference's ``PostProcessPanoptic`` (src/trackformer/models/detr_segmentation.py:256-388) on CPU, imported
as tests/golden/make_golden_model.py imports the reference (visdom and the compiled extension stubbed).  panopticapi is
not installed, so this recorder supplies ``panopticapi.utils.id2rgb`` / ``rgb2id`` itself (written from their
definition: R + 256 G + 256^2 B).  Stores tests/golden/panoptic_postprocess.npz: per case the inputs, the decoded
target-size id maps and ``segments_info`` (as JSON).

Cases: a batch of two differently sized images with stuff duplicates and the small-segment filter re-running,
everything filtered, and an image with more than 255 surviving segments (the G channel of id2rgb).  Seeds are
searched so that at every processed pixel the top two upsampled logits of the kept queries (and of the survivors) are
equal or at least 1e-3 apart, and no kept score lies within 1e-4 of the threshold: the fixtures hold no near-ties.
An image without a kept query is not recorded: the reference's ``interpolate`` of zero masks raises in current torch
(upsample_bilinear2d refuses an empty tensor); tests/test_panoptic_cpu.py checks that case by construction.
"""
import io
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def _utils():
    def id2rgb(id_map):
        if isinstance(id_map, np.ndarray):
            c = id_map.copy()
            rgb = np.zeros(tuple(id_map.shape) + (3,), np.uint8)
            for i in range(3):
                rgb[..., i] = c % 256
                c //= 256
            return rgb
        out = []
        for _ in range(3):
            out.append(id_map % 256)
            id_map //= 256
        return out

    def rgb2id(color):
        if isinstance(color, np.ndarray) and len(color.shape) == 3:
            if color.dtype == np.uint8:
                color = color.astype(np.int32)
            return color[:, :, 0] + 256 * color[:, :, 1] + 256 * 256 * color[:, :, 2]
        return int(color[0] + 256 * color[1] + 256 * 256 * color[2])
    pkg = types.ModuleType("panopticapi")
    utils = types.ModuleType("panopticapi.utils")
    utils.id2rgb, utils.rgb2id = id2rgb, rgb2id
    pkg.utils = utils
    sys.modules["panopticapi"] = pkg
    sys.modules["panopticapi.utils"] = utils


LOGIT_STEP = 0.125     # class logits are int8 multiples of this: stored as int8, exact in fp32
MASK_STEP = 2.0 ** -7  # mask logits are int16 multiples of this


def make_case(seed, B, Q, hw, sizes, tsizes, n_keep, classes, winners=False):
    """Inputs whose values are int8 multiples of LOGIT_STEP and int16 multiples of MASK_STEP, so the fixture stores
    them as those integers and the tests widen them to exactly these fp32 values.  ``winners``: every processed pixel (hw is then the processed
    size) has one kept query strictly above all others; all but three kept queries win at least two pixels, so those
    survive and the three that win nothing are filtered."""
    g = torch.Generator().manual_seed(seed)
    C = 251
    logits = (torch.randn(B, Q, C, generator=g) * 8).round().clamp(-127, 127)
    logits[..., -1] = 40.0                                      # no object by default (5.0)
    keeps = []
    for b in range(B):
        k = n_keep[b]
        q = torch.randperm(Q, generator=g)[:k]
        cls = torch.as_tensor([classes[int(i) % len(classes)] for i in torch.randint(0, 10 ** 6, (k,), generator=g)],
                              dtype=torch.long)
        logits[b, q, cls] = 120.0                               # 15.0: softmax score well above 0.85
        keeps.append(q)
    h, w = hw
    masks = torch.randint(-16256, 12801, (B, Q, h, w), generator=g).float()
    if winners:                                                 # no interpolation here: coarse losers suffice
        masks = torch.randint(-7, 8, (B, Q, h, w), generator=g).float() * 1024
        for b, q in enumerate(keeps):
            win = q[:-3]
            pix = torch.cat([win.repeat(2), win[torch.randint(0, len(win), (h * w - 2 * len(win),), generator=g)]])
            pix = pix[torch.randperm(h * w, generator=g)].view(h, w)
            masks[b].scatter_(0, pix[None], 16256.0)
    return logits * LOGIT_STEP, masks * MASK_STEP, sizes, tsizes


def gaps_ok(logits, masks, sizes, thr=0.85):
    prob = logits.softmax(-1)
    scores, labels = prob.max(-1)
    keep = labels.ne(logits.shape[-1] - 1) & (scores > thr)
    if ((scores - thr).abs() < 1e-4).any():
        return False
    for b, size in enumerate(sizes):
        m = masks[b][keep[b]]
        if len(m) < 2:
            continue
        up = F.interpolate(m[None], size=size, mode="bilinear", align_corners=False)[0]
        top = up.topk(2, dim=0).values
        d = top[0] - top[1]
        if ((d != 0) & (d < 1e-3)).any():
            return False
    return True


def main():
    _utils()
    from make_golden_model import import_reference
    import_reference()
    import trackformer.models.detr_segmentation as seg
    counter = {"n": 0}
    orig = seg.Image.fromarray

    def counting(*a, **k):
        counter["n"] += 1
        return orig(*a, **k)
    seg.Image.fromarray = counting
    is_thing_map = {i: i <= 90 for i in range(201)}
    post = seg.PostProcessPanoptic(is_thing_map, threshold=0.85)

    specs = {
        # two images, stuff duplicates (classes > 90 repeat), the small-segment filter re-running the label pass
        "batch2": dict(B=2, Q=24, hw=(24, 32), sizes=[(90, 120), (70, 110)], tsizes=[(57, 83), (140, 215)],
                       n_keep=[14, 18], classes=[1, 5, 17, 95, 120, 180], min_passes=[2, 2]),
        "all_filtered": dict(B=1, Q=20, hw=(8, 8), sizes=[(30, 30)], tsizes=[(2, 2)], n_keep=[5],
                             classes=[3, 100, 150, 7], min_passes=[2]),
        "many_kept": dict(B=1, Q=270, hw=(24, 24), sizes=[(24, 24)], tsizes=[(72, 75)], n_keep=[265], winners=True,
                          classes=list(range(1, 91)), min_passes=[2]),
    }
    out = {}
    for name, sp in specs.items():
        for seed in range(60):
            logits, masks, sizes, tsizes = make_case(seed, sp["B"], sp["Q"], sp["hw"], sp["sizes"], sp["tsizes"],
                                                     sp["n_keep"], sp["classes"], sp.get("winners", False))
            if not gaps_ok(logits, masks, sizes):
                continue
            outputs = {"pred_logits": logits, "pred_masks": masks, "pred_boxes": torch.rand(sp["B"], sp["Q"], 4)}
            preds, passes = [], []
            for b in range(sp["B"]):                          # per image, to count each image's passes
                counter["n"] = 0
                one = {k: v[b:b + 1] for k, v in outputs.items()}
                preds += post(one, [torch.tensor(sizes[b])], [torch.tensor(tsizes[b])])
                passes.append(counter["n"])
            if any(p < m for p, m in zip(passes, sp["min_passes"])):
                continue
            # the surviving queries must hold no near-ties either
            if name == "many_kept" and max(len(p["segments_info"]) for p in preds) <= 255:
                continue
            batch = post(outputs, [torch.tensor(s) for s in sizes], [torch.tensor(s) for s in tsizes])
            assert [p["segments_info"] for p in batch] == [p["segments_info"] for p in preds]
            break
        else:
            raise SystemExit(f"no seed found for {name}")
        from PIL import Image
        maps = [seg.rgb2id(np.array(Image.open(io.BytesIO(p["png_string"])), dtype=np.uint8)) for p in batch]
        print(name, "seed", seed, "passes", passes, "segments", [len(p["segments_info"]) for p in batch])
        out[f"{name}/logits"] = (logits / LOGIT_STEP).numpy().astype(np.int8)
        out[f"{name}/masks"] = (masks / MASK_STEP).numpy().astype(np.int16)
        out[f"{name}/sizes"] = np.asarray(sizes, np.int64)
        out[f"{name}/tsizes"] = np.asarray(tsizes, np.int64)
        for b, m in enumerate(maps):
            out[f"{name}/map{b}"] = m.astype(np.int16)
        out["logit_step"], out["mask_step"] = np.float32(LOGIT_STEP), np.float32(MASK_STEP)
        out[f"{name}/segments_info"] = np.frombuffer(json.dumps([p["segments_info"] for p in batch]).encode(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "panoptic_postprocess.npz"), **out)


if __name__ == "__main__":
    main()
