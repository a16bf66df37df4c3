"""Panoptic post-processing and PQ scoring on the CPU suite.

csrc/panoptic_core.h -- the routines csrc/panoptic.cu's kernels are compiled from -- is built here by g++ with one
"thread" (tests/host_build/panoptic_host.cpp, entries named like the device ones) and driven through the product's own
host code with CPU tensors: `PostProcessPanoptic.label_maps` against the reference's fixtures
(tests/golden/panoptic_postprocess.npz), and `PQScorer` / `pq_compute` against the numpy oracle
(tests/panoptic_eval_reference.py), which is first pinned on hand-worked scenes."""
import io
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import host_twin
import panoptic_eval_reference as ref
import panoptic_fixtures as pf
from trackformer_b200 import panoptic_eval as pe
from trackformer_b200.segmentation import PostProcessPanoptic

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "panoptic_postprocess.npz")
CASES = ("batch2", "all_filtered", "many_kept")
IS_THING = {i: i <= 90 for i in range(201)}


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    return pe.bind(host_twin.build("panoptic_host", tmp_path_factory.mktemp("panoptic")))


def golden_case(name):
    z = np.load(GOLDEN)
    B = len(z[f"{name}/sizes"])
    # the inputs are stored as the integers they are multiples of (make_golden_panoptic.py); fp32 holds them exactly
    logits = z[f"{name}/logits"].astype(np.float32) * np.float32(z["logit_step"])
    masks = z[f"{name}/masks"].astype(np.float32) * np.float32(z["mask_step"])
    outputs = {"pred_logits": torch.from_numpy(logits), "pred_masks": torch.from_numpy(masks)}
    sizes = [tuple(int(v) for v in s) for s in z[f"{name}/sizes"]]
    tsizes = [tuple(int(v) for v in s) for s in z[f"{name}/tsizes"]]
    maps = [z[f"{name}/map{b}"].astype(np.int32) for b in range(B)]
    infos = json.loads(bytes(z[f"{name}/segments_info"]).decode())
    return outputs, sizes, tsizes, maps, infos


@pytest.mark.parametrize("name", CASES)
def test_host_build_reproduces_reference_fixture(host_lib, name):
    outputs, sizes, tsizes, maps, infos = golden_case(name)
    post = PostProcessPanoptic(IS_THING, threshold=0.85)
    got, got_infos = post.label_maps(outputs, [torch.tensor(s) for s in sizes], [torch.tensor(s) for s in tsizes],
                                     lib=host_lib)
    assert got_infos == infos
    for m, want in zip(got, maps):
        np.testing.assert_array_equal(m.numpy(), want)


def test_fixture_cases_cover_the_issue():
    _, _, _, maps, infos = golden_case("many_kept")
    assert maps[0].max() > 255 and len(infos[0]) > 255               # the G channel of id2rgb
    _, _, _, maps, infos = golden_case("all_filtered")
    assert infos == [[]] and not maps[0].any()
    outputs, _, _, _, infos = golden_case("batch2")
    assert len(infos) == 2


def test_no_kept_query_gives_zero_map(host_lib):
    logits = torch.zeros(1, 5, 251)
    logits[..., -1] = 10.0
    outputs = {"pred_logits": logits, "pred_masks": torch.randn(1, 5, 8, 8)}
    maps, infos = PostProcessPanoptic(IS_THING).label_maps(outputs, [(30, 31)], [(20, 22)], lib=host_lib)
    assert infos == [[]] and maps[0].shape == (20, 22) and not maps[0].any()


def test_unknown_class_raises_keyerror(host_lib):
    logits = torch.zeros(1, 3, 251)
    logits[0, 0, 230] = 20.0                                          # class 230 is not in is_thing_map
    logits[0, 1:, -1] = 20.0
    with pytest.raises(KeyError):
        PostProcessPanoptic(IS_THING).label_maps({"pred_logits": logits, "pred_masks": torch.randn(1, 3, 8, 8)},
                                                 [(16, 16)], None, lib=host_lib)


def test_png_string_is_pillows_png_of_the_map():
    _, _, _, maps, _ = golden_case("many_kept")
    with io.BytesIO() as out:
        Image.fromarray(pe.id2rgb(maps[0])).save(out, format="PNG")
        want = out.getvalue()
    assert pe.png_of(maps[0]) == want
    back = pe.rgb2id(np.array(Image.open(io.BytesIO(want)), dtype=np.uint8))
    np.testing.assert_array_equal(back, maps[0])


def test_build_model_panoptic_postprocessors():
    from trackformer_b200.model_factory import build_model, vanilla_args
    from trackformer_b200.segmentation import DETRSegm, PostProcessSegm
    model, _, post = build_model(vanilla_args(masks=True, dataset="coco_panoptic", device="cpu"))
    assert type(model) is DETRSegm and model.class_embed.out_features == 251
    assert sorted(post) == ["bbox", "panoptic", "segm"] and isinstance(post["segm"], PostProcessSegm)
    pan = post["panoptic"]
    assert isinstance(pan, PostProcessPanoptic) and pan.threshold == 0.85
    assert pan.is_thing_map == {i: i <= 90 for i in range(201)}


# ---- PQ ------------------------------------------------------------------------------------------------------------
CATS = [{"id": 1, "isthing": 1}, {"id": 2, "isthing": 1}, {"id": 50, "isthing": 0}]


def _one(gt_segs, gt_map, pred_segs, pred_map, image_id=7):
    gt = {"categories": CATS, "annotations": [{"image_id": image_id, "file_name": "a.png", "segments_info": gt_segs}]}
    pr = {"annotations": [{"image_id": image_id, "file_name": "a.png", "segments_info": pred_segs}]}
    return gt, pr, {image_id: np.asarray(gt_map, np.int32)}, {image_id: np.asarray(pred_map, np.int32)}


def _gs(i, c, a, crowd=0):
    return {"id": i, "category_id": c, "area": a, "iscrowd": crowd}


def _stat(stat, c):
    s = stat[c]
    return s.tp, s.fp, s.fn, s.iou


def test_oracle_match_and_void():
    # GT 5 (cat 1) covers 6 pixels; pred 9 (cat 1) covers 4 of them and 2 VOID pixels: union = 6 + 6 - 4 - 2 = 6
    gt = [[5, 5, 5, 0, 0], [5, 5, 5, 0, 0]]
    pr = [[9, 9, 0, 9, 9], [9, 9, 0, 0, 0]]
    stat = ref.pq_stats(*_one([_gs(5, 1, 6)], gt, [{"id": 9, "category_id": 1}], pr))
    assert _stat(stat, 1) == (1, 0, 0, 4 / 6)


def test_oracle_iou_exactly_half_is_no_match():
    gt = [[5, 5, 5, 5]]
    pr = [[9, 9, 0, 0]]                                              # union 4 + 2 - 2 = 4 ... iou 2/4 = 0.5
    stat = ref.pq_stats(*_one([_gs(5, 1, 4)], gt, [{"id": 9, "category_id": 1}], pr))
    assert _stat(stat, 1) == (0, 1, 1, 0.0)


def test_oracle_crowd_and_category_mismatch():
    gt = [[5, 5, 6, 6], [5, 5, 6, 6]]
    pr = [[9, 9, 8, 8], [9, 9, 8, 8]]
    segs = [_gs(5, 1, 4), _gs(6, 2, 4, crowd=1)]
    # 9 has the wrong category for 5 (FN 5, FP 9 in cat 2); 8 lies on the crowd region of its category: not an FP
    stat = ref.pq_stats(*_one(segs, gt, [{"id": 9, "category_id": 2}, {"id": 8, "category_id": 2}], pr))
    assert _stat(stat, 1) == (0, 0, 1, 0.0) and _stat(stat, 2) == (0, 1, 0, 0.0)


def test_oracle_unlisted_gt_is_not_void():
    gt = [[5, 5, 7, 7]]                                              # 7 is not listed
    pr = [[9, 9, 9, 9]]
    stat = ref.pq_stats(*_one([_gs(5, 1, 2)], gt, [{"id": 9, "category_id": 1}], pr))
    assert _stat(stat, 1) == (0, 1, 1, 0.0)                          # union 4 + 2 - 2 = 4, iou 0.5


def test_oracle_errors():
    gt = [[5, 5]]
    with pytest.raises(KeyError, match="presented in PNG and not presented in JSON"):
        ref.pq_stats(*_one([_gs(5, 1, 2)], gt, [], [[3, 3]]))
    with pytest.raises(KeyError, match="unknown category_id 4"):
        ref.pq_stats(*_one([_gs(5, 1, 2)], gt, [{"id": 3, "category_id": 4}], [[3, 3]]))
    with pytest.raises(KeyError, match="presented in JSON and not presented in PNG"):
        ref.pq_stats(*_one([_gs(5, 1, 2)], gt, [{"id": 3, "category_id": 1}, {"id": 4, "category_id": 1}],
                             [[3, 3]]))
    g, p, gm, pm = _one([_gs(5, 1, 2)], gt, [], [[0, 0]])
    p["annotations"][0]["image_id"] = 8
    with pytest.raises(Exception, match="no prediction for the image with id: 7"):
        ref.pq_stats(g, p, gm, pm)


def host_pq(lib, gt_json, pred_json, gt_maps, pred_maps, batch=3):
    scorer = pe.PQScorer(gt_json["categories"], "cpu", lib)
    preds = {a["image_id"]: a for a in pred_json["annotations"]}
    anns = gt_json["annotations"]
    for c in range(0, len(anns), batch):
        scorer.add([dict(gt_ann=a, gt_map=gt_maps[a["image_id"]], pred_ann=preds[a["image_id"]],
                         pred_map=pred_maps[a["image_id"]]) for a in anns[c:c + batch]])
    tp, fp, fn, iou = scorer.result([a["image_id"] for a in anns])
    return pe.pq_results(scorer.cats, tp, fp, fn, iou), (tp, fp, fn, iou), scorer


def assert_results_equal(got, want):
    for name in ("All", "Things", "Stuff"):
        assert got[name]["n"] == want[name]["n"]
        for k in ("pq", "sq", "rq"):
            assert abs(got[name][k] - want[name][k]) <= 1e-12
    assert got["per_class"].keys() == want["per_class"].keys()
    for c in want["per_class"]:
        for k in ("pq", "sq", "rq"):
            assert abs(got["per_class"][c][k] - want["per_class"][c][k]) <= 1e-12


@pytest.mark.parametrize("seed", range(20))
def test_host_build_equals_oracle(host_lib, seed):
    data = pf.dataset(seed, 5)
    want, stat = ref.pq_compute(*data)
    got, (tp, fp, fn, iou), scorer = host_pq(host_lib, *data)
    for k, c in enumerate(scorer.cats.ids):
        s = stat[c]
        assert (tp[k], fp[k], fn[k]) == (s.tp, s.fp, s.fn)
        assert abs(iou[k] - s.iou) <= 1e-12
    assert_results_equal(got, want)


@pytest.mark.parametrize("case", ["unlisted", "category", "missing"])
def test_host_build_errors(host_lib, case):
    gt = [[5, 5, 5]]
    pred = {"unlisted": ([], [[3, 3, 0]]), "category": ([{"id": 3, "category_id": 4}], [[3, 3, 0]]),
            "missing": ([{"id": 3, "category_id": 1}, {"id": 4, "category_id": 1}], [[3, 3, 0]])}[case]
    data = _one([_gs(5, 1, 3)], gt, *pred)
    with pytest.raises(KeyError) as want:
        ref.pq_stats(*data)
    with pytest.raises(KeyError) as got:
        host_pq(host_lib, *data)
    assert str(got.value) == str(want.value)


def test_host_build_duplicate_image_and_size_mismatch(host_lib):
    gt_json, pred_json, gmaps, pmaps = pf.dataset(3, 2)
    scorer = pe.PQScorer(gt_json["categories"], "cpu", host_lib)
    a0 = gt_json["annotations"][0]
    empty = dict(pred_json["annotations"][0], segments_info=[])              # a first, wrong prediction ...
    scorer.add([dict(gt_ann=a0, gt_map=gmaps[a0["image_id"]], pred_ann=empty,
                     pred_map=np.zeros_like(gmaps[a0["image_id"]]))])
    preds = {a["image_id"]: a for a in pred_json["annotations"]}
    for a in gt_json["annotations"]:                                         # ... then the right one: the last wins
        scorer.add([dict(gt_ann=a, gt_map=gmaps[a["image_id"]], pred_ann=preds[a["image_id"]],
                         pred_map=pmaps[a["image_id"]])])
    got = pe.pq_results(scorer.cats, *scorer.result([a["image_id"] for a in gt_json["annotations"]]))
    assert_results_equal(got, ref.pq_compute(gt_json, pred_json, gmaps, pmaps)[0])
    with pytest.raises(ValueError, match="prediction map"):
        scorer.add([dict(gt_ann=a0, gt_map=gmaps[a0["image_id"]], pred_ann=preds[a0["image_id"]],
                         pred_map=pmaps[a0["image_id"]][:, :-1])])
    with pytest.raises(Exception, match="no prediction for the image with id: 99"):
        scorer.result([99])


def test_pq_compute_over_png_folders(host_lib, tmp_path, capsys):
    gt_json, pred_json, gmaps, pmaps = pf.dataset(11, 4)
    for side, js, maps in (("gt", gt_json, gmaps), ("pred", pred_json, pmaps)):
        d = tmp_path / side
        d.mkdir()
        for a in js["annotations"]:
            Image.fromarray(pe.id2rgb(maps[a["image_id"]])).save(d / a["file_name"])
        (tmp_path / f"{side}.json").write_text(json.dumps(js))
    got = pe.pq_compute(str(tmp_path / "gt.json"), str(tmp_path / "pred.json"), str(tmp_path / "gt"),
                        str(tmp_path / "pred"), device="cpu", lib=host_lib)
    assert_results_equal(got, ref.pq_compute(gt_json, pred_json, gmaps, pmaps)[0])
    assert "PQ     SQ     RQ     N" in capsys.readouterr().out
