"""The reference's PostProcessPanoptic restated with torch ops on any device (tests and tools/panoptic_bench.py):
kept queries by softmax, bilinear upsampling of the kept padded logits to the processed size, softmax-argmax over the
kept queries, the stuff merge on the first pass, Pillow's NEAREST resize as an index map, areas, and the small-segment
filter loop.  Returns per image (target-size map [Ht, Wt] long, segments_info, the first pass's probabilities
[K, H, W] for near-tie checks)."""
import torch
import torch.nn.functional as F

from trackformer_b200.segmentation import pillow_nearest_src


def postprocess(outputs, sizes, tsizes, is_thing_map, threshold=0.85, keep_probs=False):
    logits, masks = outputs["pred_logits"], outputs["pred_masks"]
    res = []
    for b in range(len(sizes)):
        (H, W), (Ht, Wt) = sizes[b], tsizes[b]
        scores, labels = logits[b].softmax(-1).max(-1)
        keep = labels.ne(logits.shape[-1] - 1) & (scores > threshold)
        classes = labels[keep]
        m = masks[b][keep]
        dev = m.device
        rows = torch.from_numpy(pillow_nearest_src(H, Ht)).to(dev)
        cols = torch.from_numpy(pillow_nearest_src(W, Wt)).to(dev)
        if len(m):
            m = F.interpolate(m[None], size=(H, W), mode="bilinear", align_corners=False)[0]
        stuff = {}
        for k, c in enumerate(classes.tolist()):
            if not is_thing_map[c]:
                stuff.setdefault(c, []).append(k)
        first_probs = None

        def ids_area(mk, dedup):
            nonlocal first_probs
            if len(mk) == 0:
                mid = torch.zeros((H, W), dtype=torch.long, device=dev)
            else:
                p = mk.softmax(0)
                if keep_probs and first_probs is None:
                    first_probs = p
                mid = p.argmax(0)
            if dedup:
                for eq in stuff.values():
                    for e in eq:
                        mid[mid == e] = eq[0]
            t = mid[rows][:, cols]
            return [int((t == i).sum()) for i in range(len(mk))], t
        area, t = ids_area(m, True)
        while len(classes):
            small = torch.tensor([a <= 4 for a in area], dtype=torch.bool, device=dev)
            if not small.any():
                break
            classes, m = classes[~small], m[~small]
            area, t = ids_area(m, False)
        info = [{"id": i, "isthing": is_thing_map[int(classes[i])], "category_id": int(classes[i]), "area": a}
                for i, a in enumerate(area)]
        res.append((t, info, first_probs))
    return res
