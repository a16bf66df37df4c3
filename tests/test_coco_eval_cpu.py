"""COCO evaluation on the CPU suite.

The oracle (tests/coco_eval_reference.py) is pinned on hand-worked scenes; then csrc/coco_eval_core.h -- the routines
csrc/coco_eval.cu's kernels are compiled from, built here by g++ with one "thread" (tests/host_build/coco_eval_host.cpp)
-- is compared with the oracle on seeded synthetic scenes through the product's own packing (`GroundTruth`,
`pack_update`, `kept_images`).  Also: ground-truth loading, polygon rejection, the rank gather-and-dedupe, the
`summarize()` format, the `.eval` pickle round trip and the C entries' argument checks.  The CUDA build of the same
source is compared in tests/test_coco_eval_gpu.py."""
import ctypes
import json
import os
import pickle

import numpy as np
import pytest
import torch

import coco_eval_fixtures as cf
import coco_eval_reference as ref
import host_twin
from trackformer_b200 import coco_eval as ce



@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    lib = host_twin.build("coco_eval_host", tmp_path_factory.mktemp("coco_eval"))
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    lib.tfb200_coco_match_host.argtypes = ([vp, i32, i32, i32, vp, vp, vp, i64, vp, i32] + [vp] * 11
                                           + [i32, vp, i32, i32, i32, i64, i64, i64, i64, vp, vp, vp, vp, vp])
    lib.tfb200_coco_match_host.restype = i32
    lib.tfb200_coco_accumulate_host.argtypes = ([vp, vp, vp, i64, vp, i32, i64, vp, vp, vp, vp, i32, i32, i32, i32,
                                                 i32, vp, vp, vp, vp])
    lib.tfb200_coco_accumulate_host.restype = i32
    return lib


def _p(a):
    return a.ctypes.data


def host_eval(lib, dataset, updates, iou_type, iou_out=None):
    """The device algorithm run on the host through the product's packing: (precision, recall, scores, stats).
    `iou_out` (a list) receives per update (pack_update's dict, the IoU workspace, the sort keys)."""
    segm = iou_type == "segm"
    gt = ce.GroundTruth(dataset, segm)
    params = ce.Params(iou_type, gt.cat_ids.tolist())
    A, T = len(params.areaRng), len(params.iouThrs)
    g = {k: np.ascontiguousarray(v) for k, v in gt.arrays().items()}
    dummy = np.zeros(8, np.int64)
    gp = lambda k: _p(g[k]) if k in g and g[k].size else _p(dummy)
    area_rng = np.asarray(params.areaRng, np.float64)
    iou_thr = np.minimum(params.iouThrs, 1 - 1e-10)
    status = np.zeros(1, np.int32)
    recs = []
    for upd in updates:
        ids = [int(i) for i in np.unique(list(upd.keys()))]
        z = ce.pack_update(gt, params, ids, upd, segm)
        img = z["img"]
        masks = [np.ascontiguousarray(m.numpy().astype(np.uint8)) for m in z["masks"]]
        if segm:
            img[:, 5] = [_p(m) if m.size else _p(dummy) for m in masks]
        N = z["N"]
        cat = lambda xs, dt: np.ascontiguousarray(torch.cat(xs).numpy().astype(dt)) if xs else np.zeros(0, dt)
        scores, labels = cat(z["scores"], np.float32), cat(z["labels"], np.int64)
        boxes = cat(z["boxes"], np.float32) if not segm else np.zeros(4, np.float32)
        key, rank, state = np.zeros(N, np.uint64), np.zeros(N, np.int32), np.zeros(N * A, np.uint32)
        iou = np.zeros(z["iou_cells"], np.float64)
        nz = lambda a: _p(a) if a.size else _p(dummy)
        rc = lib.tfb200_coco_match_host(
            _p(img), len(ids), z["max_n"], z["max_g"], nz(boxes), nz(scores), nz(labels), N, gp("cat_ids"),
            len(gt.cat_ids), gp("off"), gp("k"), gp("box"), gp("area"), gp("crowd"), gp("id"), gp("run_off"),
            gp("runs"), gp("bbox"), gp("px"), _p(area_rng), A, _p(iou_thr), T, params.maxDets[-1], int(segm),
            z["iou_cells"], z["dbit_words"], z["gbit_words"], z["gtm_bytes"], nz(key), nz(rank), nz(state),
            _p(status), nz(iou))
        assert rc == 0
        if iou_out is not None:
            iou_out.append((z, iou, key))
        counts = np.asarray([int(s.shape[0]) for s in z["scores"]], np.int64)
        recs.append((np.asarray(ids), counts, key, rank, state))
    ids, begins, counts = ce.kept_images([(r[0], r[1]) for r in recs])
    key = np.concatenate([r[2] for r in recs])
    rank = np.concatenate([r[3] for r in recs])
    state = np.concatenate([r[4] for r in recs])
    dst = np.concatenate(([0], np.cumsum(counts)[:-1])).astype(np.int64)
    kept = np.ascontiguousarray(np.stack((begins, dst, counts), 1).astype(np.int64))
    npig = np.ascontiguousarray(gt.npig([gt.row_of[i] for i in ids], params.areaRng))
    K, R, M = len(gt.cat_ids), len(params.recThrs), len(params.maxDets)
    precision, scores_o = np.zeros((T, R, K, A, M)), np.zeros((T, R, K, A, M))
    recall, st = np.zeros((T, K, A, M)), np.zeros(1)
    max_dets = np.asarray(params.maxDets, np.int32)
    rc = lib.tfb200_coco_accumulate_host(
        nz(key), nz(rank), nz(state), len(key), nz(kept), len(ids), int(counts.sum()), _p(npig),
        _p(np.ascontiguousarray(params.recThrs)), _p(max_dets), _p(status), K, A, T, R, M, _p(precision),
        _p(recall), _p(scores_o), _p(st))
    assert rc == 0
    params.imgIds = ids.tolist()
    stats = ce.summarize_eval({"precision": precision, "recall": recall}, params, out=lambda s: None)
    return precision, recall, scores_o, stats


# ---------------------------------------------------------------- hand-worked scenes (oracle and host build)

def _ds(anns, cats=(1,), images=((1, 100, 100),)):
    for i, a in enumerate(anns):
        a.setdefault("id", i + 1)
        a.setdefault("image_id", 1)
        a.setdefault("category_id", 1)
        a.setdefault("iscrowd", 0)
        a.setdefault("area", a["bbox"][2] * a["bbox"][3])
    return {"images": [{"id": i, "height": h, "width": w} for i, h, w in images], "annotations": anns,
            "categories": [{"id": c} for c in cats]}


def _pred(boxes, scores, labels=None):
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    n = len(boxes)
    return {"boxes": torch.from_numpy(boxes), "scores": torch.tensor(scores, dtype=torch.float32),
            "labels": torch.tensor(labels if labels is not None else [0] * n, dtype=torch.int64)}


def both(host_lib, dataset, updates, iou_type="bbox"):
    o = ref.coco_eval(dataset, cf.as_numpy(updates), iou_type)
    h = host_eval(host_lib, dataset, updates, iou_type)
    for x, y in zip(o, h):
        assert np.array_equal(x, y)
    return o


def test_crowd_ground_truth(host_lib):
    """One GT box [0, 0, 10, 10] and a crowd region [20, 0, 40, 20].  Detections: two inside the crowd region
    (IoU = area over the detection's own area = 1) and one on the GT.  The crowd matches both (matched many times)
    and both are ignored; the third is a tp.  So precision 1 at every recall threshold, AP = AR = 1."""
    ds = _ds([{"bbox": [0, 0, 10, 10]}, {"bbox": [20, 0, 20, 20], "iscrowd": 1}])
    up = [{1: _pred([[22, 2, 30, 10], [25, 5, 35, 15], [0, 0, 10, 10]], [0.9, 0.8, 0.7])}]
    p, r, s, stats = both(host_lib, ds, up)
    assert np.isclose(stats[0], 1.0) and stats[8] == 1.0
    assert np.allclose(p[:, :, 0, 0, 2], 1.0)
    # scores: recall threshold 0 takes the first detection (the ignored 0.9), the others the tp's 0.7
    assert np.all(s[:, 0, 0, 0, 2] == np.float32(0.9)) and np.all(s[:, 1:, 0, 0, 2] == np.float32(0.7))


def test_iou_exactly_at_a_threshold(host_lib):
    """GT [0, 0, 10, 10], detection [0, 0, 20, 10]: IoU = 100 / 200 = 0.5 exactly, which matches at t = 0.5 (>=)
    and at no other threshold.  AP@0.5 = 1, AP@0.75 = 0,
    AP = 1/10 = 0.1."""
    ds = _ds([{"bbox": [0, 0, 10, 10]}])
    p, r, s, stats = both(host_lib, ds, [{1: _pred([[0, 0, 20, 10]], [0.5])}])
    assert np.isclose(stats[1], 1.0) and stats[2] == 0.0 and np.isclose(stats[0], 0.1)


def test_area_exactly_32_squared_and_96_squared(host_lib):
    """GT areas 1024 and 9216 are both small and medium, and medium and large (inclusive bounds): each range has
    its GT; the matched detections (areas 1024 and 9216) are inside both of their ranges."""
    ds = _ds([{"bbox": [0, 0, 32, 32]}, {"bbox": [0, 40, 96, 96]}], images=((1, 200, 200),))
    up = [{1: _pred([[0, 0, 32, 32], [0, 40, 96, 136]], [0.9, 0.8])}]
    p, r, s, stats = both(host_lib, ds, up)
    assert np.allclose(stats[3:6], 1.0) and list(stats[9:12]) == [1.0, 1.0, 1.0]


def test_id_zero_quirk(host_lib):
    """GT id 0 and id 1, two exact detections: the one matched to id 0 counts as a false positive (accumulate tests
    the id for truth) while the GT counts as taken.  npig = 2, tp = 1: the scores sorted 0.9 (id 0, fp), 0.8 (tp):
    pr = [0, 0.5], recall 0.5; precision 0.5 up to recall 0.5, then 0.  AP = 51 * 0.5 / 101."""
    ds = _ds([{"bbox": [0, 0, 10, 10], "id": 0}, {"bbox": [50, 50, 10, 10], "id": 1}])
    up = [{1: _pred([[0, 0, 10, 10], [50, 50, 60, 60]], [0.9, 0.8])}]
    p, r, s, stats = both(host_lib, ds, up)
    assert r[0, 0, 0, 2] == 0.5 and np.isclose(stats[0], 51 * 0.5 / 101)


def test_ignore_key_is_overwritten(host_lib):
    """An annotation with "ignore": 1 but iscrowd 0 is an ordinary GT: missing it costs recall 0.5."""
    ds = _ds([{"bbox": [0, 0, 10, 10], "ignore": 1}, {"bbox": [50, 50, 10, 10]}])
    p, r, s, stats = both(host_lib, ds, [{1: _pred([[50, 50, 60, 60]], [0.9])}])
    assert stats[8] == 0.5


def test_more_than_100_detections_in_one_category(host_lib):
    """120 misses scored above one exact hit: the hit (rank 121) is cut by the 100 truncation, so AP = AR = 0."""
    ds = _ds([{"bbox": [0, 0, 10, 10]}], images=((1, 400, 400),))
    boxes = [[200 + i % 10, 200 + i // 10, 210 + i % 10, 210 + i // 10] for i in range(120)] + [[0, 0, 10, 10]]
    p, r, s, stats = both(host_lib, ds, [{1: _pred(boxes, [0.9] * 120 + [0.1])}])
    assert stats[0] == 0.0 and stats[8] == 0.0


def test_tied_scores_across_images(host_lib):
    """Two images, same score 0.5: image 1's detection is a fp, image 2's a tp.  Ties keep image-id order, so the fp
    comes first: pr = [0, 0.5]; AP = 0.5 (all recall thresholds up to 1 reach the tp at precision 0.5)."""
    ds = _ds([{"bbox": [0, 0, 10, 10], "image_id": 2}], images=((1, 100, 100), (2, 100, 100)))
    up = [{2: _pred([[0, 0, 10, 10]], [0.5]), 1: _pred([[0, 0, 10, 10]], [0.5])}]
    p, r, s, stats = both(host_lib, ds, up)
    assert np.isclose(stats[0], 0.5)


def test_category_without_ground_truth(host_lib):
    """Category 2 has no GT: its precision / recall stay -1 and are left out of the mean, so AP = 1 from category
    1 alone even though category 2 has a (false-positive) detection."""
    ds = _ds([{"bbox": [0, 0, 10, 10]}], cats=(1, 2))
    p, r, s, stats = both(host_lib, ds, [{1: _pred([[0, 0, 10, 10], [50, 50, 60, 60]], [0.9, 0.95], [0, 1])}])
    assert np.all(p[:, :, 1] == -1) and np.all(r[:, 1] == -1) and np.isclose(stats[0], 1.0)


def test_detections_only_and_ground_truth_only_images(host_lib):
    """Image 1: one GT, no detection.  Image 2: no GT, one detection (a fp).  npig = 1, no tp: AP = AR = 0."""
    ds = _ds([{"bbox": [0, 0, 10, 10]}], images=((1, 100, 100), (2, 100, 100)))
    up = [{1: _pred(np.zeros((0, 4)), []), 2: _pred([[0, 0, 10, 10]], [0.9])}]
    p, r, s, stats = both(host_lib, ds, up)
    assert stats[0] == 0.0 and stats[8] == 0.0


def test_envelope_and_zeros_past_the_last_recall(host_lib):
    """Three GTs, detections fp (0.9), tp (0.8), tp (0.7): pr = [0, 0.5, 0.667], envelope [0.667, 0.667, 0.667];
    recall reaches 2/3, so q = 2/3 for recall thresholds <= 0.66 (67 of them) and 0 past it."""
    ds = _ds([{"bbox": [0, 0, 10, 10]}, {"bbox": [20, 20, 10, 10]}, {"bbox": [40, 40, 10, 10]}])
    up = [{1: _pred([[70, 70, 80, 80], [0, 0, 10, 10], [20, 20, 30, 30]], [0.9, 0.8, 0.7])}]
    p, r, s, stats = both(host_lib, ds, up)
    q = p[0, :, 0, 0, 2]
    assert np.allclose(q[:67], 2 / 3) and np.all(q[67:] == 0) and np.all(s[0, 67:, 0, 0, 2] == 0)


def test_max_dets_1_and_10_against_100(host_lib):
    """Eleven GTs hit by eleven detections: AR@1 = 1/11, AR@10 = 10/11, AR@100 = 1."""
    anns = [{"bbox": [20 * i, 0, 10, 10]} for i in range(11)]
    ds = _ds(anns, images=((1, 100, 300),))
    boxes = [[20 * i, 0, 20 * i + 10, 10] for i in range(11)]
    p, r, s, stats = both(host_lib, ds, [{1: _pred(boxes, [1.0 - 0.01 * i for i in range(11)])}])
    assert np.isclose(stats[6], 1 / 11) and np.isclose(stats[7], 10 / 11) and stats[8] == 1.0


def test_float32_width_rounding_moves_a_pair_across_half(host_lib):
    """x0 = 29.971189498901367, x1 = 69.97119140625 (both float32): in doubles x1 - x0 = 40.0000019, but
    convert_to_xywh subtracts in float32, which rounds to 40.0 exactly.  Against GT [x0, 0, 20, 10] the IoU is
    200 / (10 w): exactly 0.5 with the float32 width (a match at t = 0.5, AP@0.5 = 1), 0.49999998 with the double
    one (no match)."""
    x0, x1 = np.float32(29.971189498901367), np.float32(69.97119140625)
    assert float(np.float32(x1 - x0)) == 40.0 and float(x1) - float(x0) > 40.0
    ds = _ds([{"bbox": [float(x0), 0, 20, 10]}])
    p, r, s, stats = both(host_lib, ds, [{1: _pred([[x0, 0, x1, 10]], [0.9])}])
    assert np.isclose(stats[1], 1.0) and stats[2] == 0.0


# ---------------------------------------------------------------- the host build against the oracle

@pytest.mark.parametrize("seed", range(12))
def test_host_build_matches_oracle_coco_like(host_lib, seed):
    ds, ups = cf.scene(seed, "coco")
    both(host_lib, ds, ups)


@pytest.mark.parametrize("seed", range(12))
def test_host_build_matches_oracle_mot_like(host_lib, seed):
    ds, ups = cf.scene(100 + seed, "mot", n_images=4)
    both(host_lib, ds, ups)


@pytest.mark.parametrize("seed", range(6))
def test_host_build_matches_oracle_masks(host_lib, seed):
    ds, ups = cf.scene(200 + seed, "coco" if seed % 2 else "mot", segm=True, n_images=3, size=(37, 70))
    both(host_lib, ds, ups, "segm")


def test_host_build_mask_iou_equals_numpy_counts(host_lib):
    """The IoU matrix of the host build (intersection popcounts over the boxes' overlap, union or the detection's
    area for a crowd) equals numpy's pixel counts for every evaluated (detection, same-category ground truth) pair,
    empty detection masks included."""
    seen = 0
    for seed in range(4):
        ds, ups = cf.scene(300 + seed, "coco" if seed % 2 else "mot", segm=True, n_images=3, size=(37, 70))
        out = []
        host_eval(host_lib, ds, ups, "segm", iou_out=out)
        gt = ce.GroundTruth(ds, True)
        for upd, (z, iou, key) in zip(ups, out):
            for b, img_id in enumerate(sorted(upd)):
                r = gt.row_of[img_id]
                rows = range(gt.off[r], gt.off[r + 1])
                anns = {a["id"]: a for a in ds["annotations"] if a["image_id"] == img_id}
                G, d0 = len(rows), int(z["img"][b, 1])
                masks = upd[img_id]["masks"].numpy()
                for j in range(int(z["img"][b, 2])):
                    k = int(key[d0 + j]) >> 32
                    if k >= len(gt.cat_ids):
                        continue                                   # not evaluated
                    for g, row in enumerate(rows):
                        if gt.k[row] != k:
                            continue
                        a = anns[int(gt.id[row])]
                        want = ref.mask_iou(masks[j, 0] > 0.5, ref._gt_mask(a, 37, 70), a["iscrowd"])
                        assert iou[int(z["img"][b, 6]) + j * G + g] == want
                        seen += 1
    assert seen > 100


def test_integer_masks_are_thresholded():
    """Masks of a dtype other than bool / uint8 are taken as `masks > 0.5`, as the reference does, so an int64 0/1
    mask packs like its bool copy (the kernel reads one byte per pixel)."""
    ds, ups = cf.scene(5, "coco", segm=True, n_images=2, size=(20, 30), updates=1)
    gt = ce.GroundTruth(ds, True)
    params = ce.Params("segm", gt.cat_ids.tolist())
    ids = sorted(ups[0])
    as_i64 = {i: dict(p, masks=p["masks"].to(torch.int64) * 3 - 1) for i, p in ups[0].items()}
    za = ce.pack_update(gt, params, ids, ups[0], True)
    zb = ce.pack_update(gt, params, ids, as_i64, True)
    for a, b in zip(za["masks"], zb["masks"]):
        assert b.dtype == torch.bool and torch.equal(a, b)


# ---------------------------------------------------------------- host-side pieces

def test_ground_truth_from_path_dict_and_dataset_object(tmp_path):
    ds, _ = cf.scene(3)
    path = tmp_path / "gt.json"
    path.write_text(json.dumps(ds))

    class Coco:
        dataset = ds

    a, b, c = (ce.GroundTruth(ce.load_dataset(x), False) for x in (str(path), ds, Coco()))
    for k in a.arrays():
        assert np.array_equal(a.arrays()[k], b.arrays()[k]) and np.array_equal(a.arrays()[k], c.arrays()[k])
    with pytest.raises(TypeError):
        ce.load_dataset(42)


def test_polygon_segmentation_is_rejected():
    ds = _ds([{"bbox": [0, 0, 10, 10], "segmentation": [[0, 0, 10, 0, 10, 10]], "id": 7}])
    with pytest.raises(NotImplementedError, match="annotation 7"):
        ce.GroundTruth(ds, True)
    ce.GroundTruth(ds, False)                        # boxes need no masks


def test_gather_and_dedupe_across_two_ranks():
    """Rank 0 evaluated images 1, 3 then 5 (padding duplicate: 1), rank 1 images 2, 4 then 1: the first record of
    each image id is kept, in image-id order."""
    r0 = [(np.array([1, 3]), np.array([2, 3])), (np.array([1, 5]), np.array([4, 1]))]
    r1 = [(np.array([2, 4]), np.array([1, 1])), (np.array([1]), np.array([7]))]
    ids, begins, counts = ce.kept_images(r0 + r1)
    assert ids.tolist() == [1, 2, 3, 4, 5]
    assert begins.tolist() == [0, 10, 2, 11, 9]
    assert counts.tolist() == [2, 1, 3, 1, 1]
    merged = ref.merge([{1: "a", 3: "b"}, {1: "c", 5: "d"}, {2: "e", 4: "f"}, {1: "g"}])
    assert merged == {1: "a", 2: "e", 3: "b", 4: "f", 5: "d"}


def test_summarize_format_and_eval_pickle():
    p = ce.Params("bbox", [1])
    ev = ce.eval_dict(p, np.full((10, 101, 1, 4, 3), 0.5), np.full((10, 1, 4, 3), 0.25),
                      np.zeros((10, 101, 1, 4, 3)))
    lines = []
    stats = ce.summarize_eval(ev, p, out=lines.append)
    assert lines[0] == " Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 0.500"
    assert lines[1] == " Average Precision  (AP) @[ IoU=0.50      | area=   all | maxDets=100 ] = 0.500"
    assert lines[6] == " Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets=  1 ] = 0.250"
    assert lines[9] == " Average Recall     (AR) @[ IoU=0.50:0.95 | area= small | maxDets=100 ] = 0.250"
    assert len(lines) == 12 and stats.dtype == np.float64 and stats.shape == (12,)
    back = pickle.loads(pickle.dumps(ev))
    assert back["counts"] == [10, 101, 1, 4, 3] and np.array_equal(back["precision"], ev["precision"])
    assert back["params"].iouType == "bbox" and back["params"].maxDets == [1, 10, 100]


def test_invalid_iou_types():
    with pytest.raises(ValueError):
        ce.CocoEvaluator({"images": [], "annotations": [], "categories": [{"id": 1}]}, ("keypoints",))


def test_c_entry_argument_checks():
    from trackformer_b200 import ext
    if not os.path.exists(ext.library_path()):
        pytest.skip("native library not built")
    lib = ce._library()
    assert lib.tfb200_coco_match_workspace_bytes(-1, 0, 0, 0, 0) == 0
    assert lib.tfb200_coco_accumulate_workspace_bytes(-1) == 0
    buf = (ctypes.c_char * 4096)()
    a = ctypes.addressof(buf)
    # NULL pointers
    assert lib.tfb200_coco_match_f32(None, 1, 0, 0, a, a, a, 0, a, 1, *[a] * 11, 4, a, 10, 100, 0, 0, 0, 0, 0, a,
                                     4096, a, a, a, a, None) == -1
    # bad sizes: B = 0, A = 9, T = 17, too many detections for one image
    for B, A, T, max_n in ((0, 4, 10, 0), (1, 9, 10, 0), (1, 4, 17, 0), (1, 4, 10, ce.MAX_DETS_PER_IMAGE + 1)):
        assert lib.tfb200_coco_match_f32(a, B, max_n, 0, a, a, a, 0, a, 1, *[a] * 11, A, a, T, 100, 0, 0, 0, 0, 0,
                                         a, 4096, a, a, a, a, None) == -2
    assert lib.tfb200_coco_accumulate_f32(a, a, a, 0, a, 0, 0, a, a, a, a, 1, 4, 10, 2000, 3, a, 4096, a, a, a, a,
                                          None) == -2
    assert lib.tfb200_coco_accumulate_f32(a, a, a, 0, a, 0, 1, a, a, a, a, 1, 4, 10, 101, 3, a, 4096, a, a, a, a,
                                          None) == -2                                    # n > n_rec
