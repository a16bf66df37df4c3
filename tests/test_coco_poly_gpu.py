"""Polygon masks on the H100: csrc/coco_poly.cu against the host build of the same source and the oracle of
tests/coco_poly_reference.py, run for run; a COCO-val-sized ground truth against the host build; `CocoEvaluator` on
polygon ground truth against the same dataset with every polygon replaced by the oracle's RLE (and against
tests/coco_eval_reference.py); integer-rectangle polygons under segm against their boxes under bbox; and
`convert_coco_poly_to_mask` against the oracle's decode + any."""
import copy

import numpy as np
import pytest
import torch

import coco_eval_fixtures as cf
import coco_eval_reference as cref
import coco_poly_fixtures as pf
import coco_poly_reference as ref
import eval_consistency_fixtures as ef
import test_eval_consistency_cpu as rel
from test_coco_eval_gpu import gpu_eval
from test_coco_poly_cpu import host_lib, host_runs  # noqa: F401  (host_lib: the module fixture)
from test_eval_consistency_gpu import CudaBackend
from trackformer_b200 import coco_eval, coco_masks, mots

pytestmark = pytest.mark.gpu


def _device_runs(segs, hw):
    return coco_masks.poly_runs(segs, hw, [f"annotation {i}" for i in range(len(segs))], "cuda")


@pytest.mark.parametrize("h,w,n,n_oracle", [(480, 640, 4000, 300), (1080, 1920, 3000, 60)])
def test_device_equals_host_build_and_oracle(cuda_device, host_lib, h, w, n, n_oracle):
    segs = pf.segmentations(h + n, n, h, w)
    if h == 1080:
        segs = pf.fma_polygons() + segs
    hw = [(h, w)] * len(segs)
    off, runs = _device_runs(segs, hw)
    h_off, h_runs, _ = host_runs(host_lib, segs, hw)
    assert np.array_equal(off, h_off) and np.array_equal(runs, h_runs)
    for a in range(n_oracle):
        assert np.array_equal(runs[off[a]:off[a + 1]], ref.ann_runs(segs[a], h, w)), a
    again = _device_runs(segs, hw)
    assert np.array_equal(again[0], off) and np.array_equal(again[1], runs)


def test_coco_val_sized_ground_truth_equals_host_build(cuda_device, host_lib):
    ds = pf.coco_val_like(0)
    gt = coco_eval.GroundTruth(ds, True, cuda_device)
    rows = [a for a in ds["annotations"]]                 # one category order per image: compare per annotation id
    by_id = {int(i): r for r, i in enumerate(gt.id)}
    hw = [(ds["images"][a["image_id"] - 1]["height"], ds["images"][a["image_id"] - 1]["width"]) for a in rows]
    h_off, h_runs, sizes = host_runs(host_lib, [a["segmentation"] for a in rows], hw)
    assert len(rows) > 30000 and sizes[0] > 10 ** 7
    for j, a in enumerate(rows):
        r = by_id[a["id"]]
        assert np.array_equal(gt.runs[gt.run_off[r]:gt.run_off[r + 1]].astype(np.int64),
                              h_runs[h_off[j]:h_off[j + 1]])


def _polygon_scene(seed):
    """cf.scene's mask scene with every GT mask replaced by a polygon inside its box (some with a second part, some
    a box list); the RLE twin has the oracle's RLE of each polygon, list counts and strings alternating."""
    ds, ups = cf.scene(300 + seed, "coco" if seed % 2 else "mot", segm=True, n_images=4, size=(37, 70))
    rng = np.random.default_rng(seed)
    poly, rle = copy.deepcopy(ds), copy.deepcopy(ds)
    hw = {im["id"]: (im["height"], im["width"]) for im in ds["images"]}
    for k, (pa, ra) in enumerate(zip(poly["annotations"], rle["annotations"])):
        x, y, bw, bh = pa["bbox"]
        n = int(rng.integers(6, 20))
        ang = np.sort(rng.uniform(0, 2 * np.pi, n))
        pts = np.stack((x + bw / 2 * (1 + np.cos(ang)), y + bh / 2 * (1 + np.sin(ang))), 1)
        seg = [[float(v) for v in np.round(pts, 2).reshape(-1)]]
        if k % 5 == 1:
            seg.append(pf._part(rng, *hw[pa["image_id"]], "star"))
        elif k % 7 == 3:
            seg = [[x, y, bw, bh]]
        pa["segmentation"] = seg
        m = ref.ann_mask(seg, *hw[pa["image_id"]])
        counts = ref.encode(m)
        ra["segmentation"] = {"size": list(hw[pa["image_id"]]),
                              "counts": counts if k % 2 else mots.encode(m)["counts"].decode()}
    return poly, rle, ups


@pytest.mark.parametrize("seed", range(4))
def test_evaluator_polygons_equal_their_rles_and_the_oracle(cuda_device, seed):
    poly, rle, ups = _polygon_scene(seed)
    a = gpu_eval(poly, ups, "segm")
    b = gpu_eval(rle, ups, "segm")
    o = cref.coco_eval(rle, cf.as_numpy(ups), "segm")
    for x, y, z in zip(a, b, o):
        assert np.array_equal(x, y) and np.array_equal(x, z)
    assert a[3][0] > 0


@pytest.mark.parametrize("seed", range(2))
def test_integer_rectangle_polygons_score_like_their_boxes(cuda_device, seed):
    ds, up = ef.coco_scene(seed)
    poly = copy.deepcopy(ds)
    for a in poly["annotations"]:
        x, y, bw, bh = a["bbox"]
        a["segmentation"] = [[x, y, x + bw, y, x + bw, y + bh, x, y + bh]]
    backend = CudaBackend()
    rel.same(backend.coco(ds, [up], "bbox"), backend.coco(poly, [up], "segm"))


def test_convert_coco_poly_to_mask_equals_oracle(cuda_device):
    rng = np.random.default_rng(9)
    h, w = 480, 640
    segs = pf.segmentations(5, 12, h, w) + [[[10.5, 20, 100, 50]], [[0, 0, 30, 40], [300, 200, 50.5, 70]]]
    dense = [rng.random((h, w)) < 0.3, np.zeros((h, w), bool), np.ones((h, w), bool)]
    segs += [mots.encode(m) for m in dense]
    segs[-1]["counts"] = segs[-1]["counts"].decode()      # str and bytes counts
    out = coco_masks.convert_coco_poly_to_mask(segs, h, w)
    want = [ref.ann_mask(s, h, w) for s in segs[:-3]] + [m.astype(np.uint8) for m in dense]
    assert out.dtype == torch.uint8 and out.device.type == "cuda"
    assert torch.equal(out.cpu(), torch.from_numpy(np.stack(want)))
    for fma in pf.fma_polygons():
        assert torch.equal(coco_masks.convert_coco_poly_to_mask([fma], 1080, 1920).cpu()[0],
                           torch.from_numpy(ref.ann_mask(fma, 1080, 1920)))
    empty = coco_masks.convert_coco_poly_to_mask([], h, w)
    assert empty.shape == (0, h, w) and empty.dtype == torch.uint8
    with pytest.raises(ValueError, match="compressed"):
        coco_masks.convert_coco_poly_to_mask([{"size": [h, w], "counts": [0, h * w]}], h, w)
    with pytest.raises(ValueError, match="segmentation 1: a malformed"):
        coco_masks.convert_coco_poly_to_mask([segs[0], {"size": [h, w], "counts": "0Y"}], h, w)
    with pytest.raises(ValueError, match="segmentation 0 has a non-finite"):
        coco_masks.convert_coco_poly_to_mask([[[0, 0, 5, float("nan"), 5, 5]]], h, w)


def test_evaluator_names_a_bad_polygon(cuda_device):
    ds = {"images": [{"id": 1, "height": 10, "width": 10}], "categories": [{"id": 1}],
          "annotations": [{"id": 3, "image_id": 1, "category_id": 1, "area": 16.0, "bbox": [1, 1, 4, 4],
                           "segmentation": [[1, 1, 5, 1, float("inf"), 5]]}]}
    with pytest.raises(ValueError, match="annotation 3 has a non-finite"):
        coco_eval.CocoEvaluator(ds, ["segm"])
