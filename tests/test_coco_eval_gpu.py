"""COCO evaluation on the GPU: `CocoEvaluator` (csrc/coco_eval.cu) against the oracle of tests/coco_eval_reference.py,
box and mask, on the seeded scenes of the CPU suite and on 1080 x 1920 mask scenes; repeatability; the per-image
limits; `PostProcessSegm(masks_on_device=True)`; and a segmentation model's own post-processed outputs fed to
`update` unchanged."""
import numpy as np
import pytest
import torch

import coco_eval_fixtures as cf
import coco_eval_reference as ref
from trackformer_b200 import coco_eval as ce
from trackformer_b200 import mots

pytestmark = pytest.mark.gpu


def _to(updates, device):
    return [{i: {k: v.to(device) for k, v in p.items()} for i, p in u.items()} for u in updates]


def gpu_eval(dataset, updates, iou_type, device="cuda"):
    ev = ce.CocoEvaluator(dataset, (iou_type,))
    for u in _to(updates, device):
        ev.update(u)
    ev.synchronize_between_processes()
    ev.accumulate()
    ev.summarize()
    e = ev.coco_eval[iou_type]
    return e.eval["precision"], e.eval["recall"], e.eval["scores"], e.stats


def check(dataset, updates, iou_type):
    o = ref.coco_eval(dataset, cf.as_numpy(updates), iou_type)
    g = gpu_eval(dataset, updates, iou_type)
    for x, y in zip(o, g):
        assert np.array_equal(x, y)
    return g


@pytest.mark.parametrize("seed", range(10))
def test_boxes_match_oracle(seed):
    ds, ups = cf.scene(seed, "coco" if seed % 2 else "mot", n_images=5)
    check(ds, ups, "bbox")


@pytest.mark.parametrize("seed", range(6))
def test_masks_match_oracle(seed):
    ds, ups = cf.scene(200 + seed, "coco" if seed % 2 else "mot", segm=True, n_images=3, size=(37, 70))
    check(ds, ups, "segm")


def test_host_tensors_and_repeatability():
    ds, ups = cf.scene(7, "coco")
    a = gpu_eval(ds, ups, "bbox", device="cpu")
    b = gpu_eval(ds, ups, "bbox")
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


def _big_mask_scene(seed):
    """1080 x 1920: rectangles, ellipses and random blobs; empty predicted masks; a crowd RLE ground truth."""
    rng = np.random.default_rng(seed)
    h, w = 1080, 1920
    yy, xx = np.mgrid[0:h, 0:w]
    images, anns, ups = [], [], {}
    for i in range(2):
        images.append({"id": i + 1, "height": h, "width": w})
        gts = []
        for j in range(6):
            cx, cy = rng.integers(100, w - 100), rng.integers(100, h - 100)
            rx, ry = rng.integers(20, 200), rng.integers(20, 300)
            kind = j % 3
            if kind == 0:
                m = (np.abs(xx - cx) <= rx) & (np.abs(yy - cy) <= ry)
            elif kind == 1:
                m = ((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 <= 1
            else:
                m = (((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 <= 1) & (rng.random((h, w)) < 0.6)
            gts.append(m)
            rle = mots.encode(m)
            rle["counts"] = rle["counts"].decode()
            anns.append({"id": len(anns), "image_id": i + 1, "category_id": 1, "segmentation": rle,
                         "area": float(m.sum()), "iscrowd": int(j == 5), "bbox": [0, 0, 1, 1]})
        n = 12
        masks = np.zeros((n, 1, h, w), bool)
        for d in range(n):
            if d < len(gts) and d % 4 != 3:
                g = gts[d]
                shift = int(rng.integers(-15, 16))
                masks[d, 0] = np.roll(g, shift, axis=1)
            elif d % 4 == 3:
                continue                                               # empty
            else:
                cx, cy = rng.integers(100, w - 100), rng.integers(100, h - 100)
                masks[d, 0] = ((xx - cx) / 80.0) ** 2 + ((yy - cy) / 120.0) ** 2 <= 1
        ups[i + 1] = {"scores": torch.from_numpy(rng.random(n).astype(np.float32)),
                      "labels": torch.zeros(n, dtype=torch.int64), "boxes": torch.zeros(n, 4),
                      "masks": torch.from_numpy(masks)}
    return {"images": images, "annotations": anns, "categories": [{"id": 1}]}, [ups]


def test_full_size_masks_match_oracle():
    ds, ups = _big_mask_scene(0)
    check(ds, ups, "segm")


def test_detections_per_image_limit():
    lim = ce.MAX_DETS_PER_IMAGE
    ds = {"images": [{"id": 1, "height": 64, "width": 64}],
          "annotations": [{"id": 1, "image_id": 1, "category_id": 1, "bbox": [0, 0, 10, 10], "area": 100.0}],
          "categories": [{"id": 1}]}
    rng = np.random.default_rng(0)

    def pred(n):
        xy = rng.integers(0, 50, (n, 2)).astype(np.float32)
        boxes = np.concatenate([xy, xy + 10], 1)
        return {"scores": torch.from_numpy(rng.random(n).astype(np.float32)),
                "labels": torch.zeros(n, dtype=torch.int64), "boxes": torch.from_numpy(boxes)}

    check(ds, [{1: pred(lim)}], "bbox")
    with pytest.raises(ValueError, match="over the limit"):
        ce.CocoEvaluator(ds, ("bbox",)).update({1: pred(lim + 1)})


def test_ground_truths_per_image_category_limit():
    lim = ce.MAX_GT_PER_IMAGE_CATEGORY

    def ds(n):
        return {"images": [{"id": 1, "height": 64, "width": 64}],
                "annotations": [{"id": i + 1, "image_id": 1, "category_id": 1, "bbox": [i % 50, i // 100, 10, 10],
                                 "area": 100.0} for i in range(n)], "categories": [{"id": 1}]}

    boxes = torch.tensor([[0, 0, 10, 10], [5, 5, 15, 15]], dtype=torch.float32)
    check(ds(lim), [{1: {"scores": torch.tensor([0.9, 0.8]), "labels": torch.zeros(2, dtype=torch.int64),
                         "boxes": boxes}}], "bbox")
    with pytest.raises(ValueError, match="ground truths of one category"):
        ce.CocoEvaluator(ds(lim + 1), ("bbox",))


def test_non_finite_score_raises_at_accumulate():
    ds, ups = cf.scene(1, "coco", updates=1)
    img = next(iter(ups[0]))
    while len(ups[0][img]["scores"]) == 0:
        ups[0].pop(img)
        img = next(iter(ups[0]))
    ups[0][img]["scores"][0] = float("nan")
    ev = ce.CocoEvaluator(ds, ("bbox",))
    ev.update(_to(ups, "cuda")[0])
    ev.synchronize_between_processes()
    with pytest.raises(ValueError, match="non-finite"):
        ev.accumulate()
    with pytest.raises(ValueError, match="non-finite"):
        ce.CocoEvaluator(ds, ("bbox",)).update(ups[0])


def test_post_process_segm_masks_on_device():
    from trackformer_b200.segmentation import PostProcessSegm
    g = torch.Generator().manual_seed(0)
    pm = (torch.randn(2, 20, 1, 24, 32, generator=g) * 4).cuda()
    sizes, orig = torch.tensor([[24, 30], [20, 32]]), torch.tensor([[50, 61], [41, 70]])
    post = PostProcessSegm()
    a = post([{}, {}], {"pred_masks": pm}, orig, sizes)
    b = post([{}, {}], {"pred_masks": pm}, orig, sizes, masks_on_device=True)
    for x, y in zip(a, b):
        assert y["masks"].is_cuda and y["masks"].dtype == torch.bool
        assert torch.equal(x["masks"].bool(), y["masks"].cpu())
    # the device masks go straight into the evaluator
    ds = {"images": [{"id": 1, "height": 50, "width": 61}], "categories": [{"id": 1}],
          "annotations": [{"id": 1, "image_id": 1, "category_id": 1, "area": 100.0, "bbox": [0, 0, 1, 1],
                           "segmentation": {"size": [50, 61], "counts": [500, 100, 50 * 61 - 600]}}]}
    n = b[0]["masks"].shape[0]
    pred = {"scores": torch.linspace(0.1, 0.9, n, device="cuda"), "labels": torch.zeros(n, dtype=torch.int64,
                                                                                          device="cuda"),
            "masks": b[0]["masks"]}
    check(ds, [{1: pred}], "segm")


def test_end_to_end_model_outputs_into_update(cuda_device):
    """DeformableDETRSegm (canonical weights) on a two-image batch, its own post-processors as `make_results` runs
    them (`DeformablePostProcess`, whose scores and boxes are strided views of one [Q, 6] row block, then
    `PostProcessSegm(masks_on_device=True)`), fed to `update` as they are.  Box and mask AP equal the oracle fed the
    same predictions `.cpu()`; the caller's labels are left as they were; the device masks equal the default route's.
    The ground truth copies some of the model's top boxes (rounded) so that matches occur."""
    import model_fixtures as mf
    from trackformer_b200.model_factory import build_model, default_args
    dev = cuda_device
    torch.manual_seed(0)
    model, _, posts = build_model(default_args(device=str(dev), masks=True))
    mf.canonical_weights_(model, 0)
    model.to(dev).eval()
    sizes, orig = [(160, 224), (128, 192)], [(80, 112), (64, 96)]
    size_t, orig_t = torch.tensor(sizes, device=dev), torch.tensor(orig, device=dev)
    with torch.no_grad():
        out, *_ = model(mf.make_images(1, sizes, dev))
        results = posts["segm"](posts["bbox"](out, orig_t), out, orig_t, size_t, masks_on_device=True)
        default = posts["segm"](posts["bbox"](out, orig_t), out, orig_t, size_t)
    for r, d in zip(results, default):
        assert r["masks"].is_cuda and r["masks"].dtype == torch.bool
        assert torch.equal(d["masks"].bool(), r["masks"].cpu())
    img_ids = [7, 9]
    host = {i: {k: v.cpu().numpy() for k, v in r.items()} for i, r in zip(img_ids, results)}
    images, anns = [], []
    for i, (h, w) in zip(img_ids, orig):
        images.append({"id": i, "height": h, "width": w})
        p = host[i]
        for q in np.argsort(-p["scores"], kind="stable")[:6]:
            x0, y0, x1, y1 = np.clip(np.round(p["boxes"][q]), 0, [w, h, w, h]).astype(int)
            if x1 - x0 < 2 or y1 - y0 < 2:
                continue
            m = np.zeros((h, w), bool)
            m[y0:y1, x0:x1] = True
            rle = mots.encode(m)
            rle["counts"] = rle["counts"].decode()
            anns.append({"id": len(anns), "image_id": i, "category_id": int(p["labels"][q]) + 1,
                         "bbox": [float(x0), float(y0), float(x1 - x0), float(y1 - y0)], "area": float(m.sum()),
                         "iscrowd": int(len(anns) == 1), "segmentation": rle})
    ds = {"images": images, "annotations": anns, "categories": [{"id": c} for c in range(1, 92)]}
    assert len(anns) >= 4
    labels_before = [r["labels"].clone() for r in results]
    ev = ce.CocoEvaluator(ds, ("bbox", "segm"))
    ev.update(dict(zip(img_ids, results)))
    ev.synchronize_between_processes()
    ev.accumulate()
    ev.summarize()
    for r, lb in zip(results, labels_before):
        assert torch.equal(r["labels"], lb)
    for t in ("bbox", "segm"):
        p, r, s, stats = ref.coco_eval(ds, [host], t)
        e = ev.coco_eval[t]
        assert np.array_equal(p, e.eval["precision"]) and np.array_equal(r, e.eval["recall"])
        assert np.array_equal(s, e.eval["scores"]) and np.array_equal(stats, e.stats)
    assert ev.coco_eval["bbox"].stats[1] > 0
