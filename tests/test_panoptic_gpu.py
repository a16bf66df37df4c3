"""Panoptic post-processing and PQ scoring on the GPU (csrc/panoptic.cu): the reference's fixtures exactly, random
logits at 800 x 1066 -> 480 x 640 against the torch restatement (differing pixels only at near-ties), PQ through
`PanopticEvaluator` (device maps) and `pq_compute` (PNG folders) against the numpy oracle, repeatability, a vanilla
DETRSegm panoptic model's own outputs, and the error cases."""
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import panoptic_eval_reference as ref
import panoptic_fixtures as pf
import panoptic_restatement as rs
from test_panoptic_cpu import CASES, IS_THING, assert_results_equal, golden_case
from trackformer_b200 import panoptic_eval as pe
from trackformer_b200.segmentation import PostProcessPanoptic

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("name", CASES)
def test_kernels_equal_reference_fixture(name):
    outputs, sizes, tsizes, maps, infos = golden_case(name)
    outputs = {k: v.to(DEV) for k, v in outputs.items()}
    preds = PostProcessPanoptic(IS_THING, maps_on_device=True)(outputs, [torch.tensor(s) for s in sizes],
                                                                [torch.tensor(s) for s in tsizes])
    assert [p["segments_info"] for p in preds] == infos
    for p, want in zip(preds, maps):
        assert p["label_map"].device.type == "cuda" and p["label_map"].dtype == torch.int32
        np.testing.assert_array_equal(p["label_map"].cpu().numpy(), want)
        assert p["png_string"] == pe.png_of(want)


def _random_outputs(seed, B=2, Q=100, hw=(200, 304), n_keep=30):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, Q, 251, generator=g)
    for b in range(B):
        q = torch.randperm(Q, generator=g)[:n_keep]
        logits[b, q, torch.randint(1, 201, (n_keep,), generator=g)] += 12.0
    masks = torch.randn(B, Q, *hw, generator=g) * 3
    return {"pred_logits": logits.to(DEV), "pred_masks": masks.to(DEV)}


def test_random_logits_differ_only_at_near_ties():
    outputs = _random_outputs(0)
    sizes, tsizes = [(800, 1066), (790, 1050)], [(480, 640), (480, 640)]
    maps, infos = PostProcessPanoptic(IS_THING).label_maps(outputs, sizes, tsizes)
    want = rs.postprocess(outputs, sizes, tsizes, IS_THING, keep_probs=True)
    total = 0
    for b, (m, (t, info, probs)) in enumerate(zip(maps, want)):
        assert [s["category_id"] for s in infos[b]] == [s["category_id"] for s in info]
        diff = (m.long() != t).nonzero()
        total += len(diff)
        if len(diff):
            rows = torch.from_numpy(rs.pillow_nearest_src(sizes[b][0], tsizes[b][0])).to(DEV)
            cols = torch.from_numpy(rs.pillow_nearest_src(sizes[b][1], tsizes[b][1])).to(DEV)
            p = probs[:, rows[diff[:, 0]], cols[diff[:, 1]]]
            top = p.topk(2, dim=0).values
            ulp = torch.nextafter(top[0], torch.full_like(top[0], 2.0)) - top[0]
            assert ((top[0] - top[1]) <= 4 * ulp).all()
    print(f"[panoptic] {total} of {2 * 480 * 640} pixels differ from the torch restatement, all at near-ties")


def _write_folder(d, js, maps):
    d.mkdir()
    for a in js["annotations"]:
        Image.fromarray(pe.id2rgb(maps[a["image_id"]])).save(d / a["file_name"])


def _scenes(tmp_path, data):
    gt_json, pred_json, gmaps, pmaps = data
    _write_folder(tmp_path / "gt", gt_json, gmaps)
    (tmp_path / "gt.json").write_text(json.dumps(gt_json))
    return tmp_path / "gt.json", tmp_path / "gt"


@pytest.mark.parametrize("seed", range(5))
def test_evaluator_from_device_maps_equals_oracle(tmp_path, seed):
    data = pf.dataset(seed, 6)
    gt_json, pred_json, gmaps, pmaps = data
    gj, gf = _scenes(tmp_path, data)
    ev = pe.PanopticEvaluator(str(gj), str(gf), output_dir=str(tmp_path / "out"))
    anns = pred_json["annotations"]
    for c in range(0, len(anns), 2):
        preds = [dict(a, png_string=pe.png_of(pmaps[a["image_id"]]),
                      label_map=torch.from_numpy(pmaps[a["image_id"]]).to(DEV)) for a in anns[c:c + 2]]
        ev.update(preds)
    ev.synchronize_between_processes()
    got = ev.summarize()
    assert_results_equal(got, ref.pq_compute(*data)[0])
    # the PNG folder and predictions.json it wrote score the same through pq_compute
    again = pe.pq_compute(str(gj), str(tmp_path / "out" / "predictions.json"), str(gf), str(tmp_path / "out"))
    assert again == got


def test_pq_compute_1080p_and_repeatable(tmp_path):
    data = pf.dataset(77, 3, H=1080, W=1920, n_gt=40, n_pred=60)
    gt_json, pred_json, gmaps, pmaps = data
    gj, gf = _scenes(tmp_path, data)
    _write_folder(tmp_path / "pred", pred_json, pmaps)
    (tmp_path / "pred.json").write_text(json.dumps(pred_json))
    a = pe.pq_compute(str(gj), str(tmp_path / "pred.json"), str(gf), str(tmp_path / "pred"))
    b = pe.pq_compute(str(gj), str(tmp_path / "pred.json"), str(gf), str(tmp_path / "pred"))
    assert a == b
    assert_results_equal(a, ref.pq_compute(*data)[0])


def test_postprocess_repeatable():
    outputs = _random_outputs(1)
    post = PostProcessPanoptic(IS_THING)
    m1, i1 = post.label_maps(outputs, [(800, 1066)] * 2, [(480, 640)] * 2)
    m2, i2 = post.label_maps(outputs, [(800, 1066)] * 2, [(480, 640)] * 2)
    assert i1 == i2 and all(torch.equal(x, y) for x, y in zip(m1, m2))


def test_detr_segm_panoptic_model_outputs_into_update(tmp_path):
    from trackformer_b200.model_factory import build_model, vanilla_args
    from trackformer_b200.util import NestedTensor
    torch.manual_seed(0)
    model, _, post = build_model(vanilla_args(masks=True, dataset="coco_panoptic"))
    model.to(DEV).eval()
    with torch.no_grad():
        model.class_embed.bias[:] = -10.0
        model.class_embed.bias[[3, 120]] = 30.0                     # some queries above the 0.85 threshold
        x = torch.randn(1, 3, 256, 320, device=DEV)
        out, *_ = model(NestedTensor(x, torch.zeros(1, 256, 320, dtype=torch.bool, device=DEV)))
    pan = post["panoptic"]
    pan.maps_on_device = True
    preds = pan(out, torch.tensor([[256, 320]]), torch.tensor([[200, 250]]))
    m = preds[0]["label_map"].cpu().numpy()
    info = preds[0]["segments_info"]
    cats = [{"id": c, "isthing": int(c <= 90)} for c in range(1, 201)]
    gmap = np.ones_like(m)
    gmap[:, 125:] = 2                                              # a thing and a stuff segment: both groups scored
    gt_ann = {"image_id": 1, "file_name": "000000000001.png",
              "segments_info": [{"id": 1, "category_id": 3, "area": int((gmap == 1).sum()), "iscrowd": 0},
                                {"id": 2, "category_id": 120, "area": int((gmap == 2).sum()), "iscrowd": 0}]}
    (tmp_path / "gt").mkdir()
    Image.fromarray(pe.id2rgb(gmap)).save(tmp_path / "gt" / gt_ann["file_name"])
    (tmp_path / "gt.json").write_text(json.dumps({"categories": cats, "annotations": [gt_ann]}))
    ev = pe.PanopticEvaluator(str(tmp_path / "gt.json"), str(tmp_path / "gt"), output_dir=str(tmp_path / "out"))
    preds[0].update(image_id=1, file_name=gt_ann["file_name"])
    pred_ann = {"image_id": 1, "file_name": gt_ann["file_name"], "segments_info": info}
    ev.update(preds)
    got = ev.summarize()
    want = ref.pq_compute({"categories": cats, "annotations": [gt_ann]}, {"annotations": [pred_ann]},
                          {1: gmap}, {1: m})[0]
    assert_results_equal(got, want)


@pytest.mark.parametrize("case", ["unlisted", "category", "missing", "no_prediction", "size"])
def test_errors_raise_without_device_fault(tmp_path, case):
    cats = [{"id": 1, "isthing": 1}]
    gt_map = np.full((4, 6), 5, np.int32)
    gt_ann = {"image_id": 7, "file_name": "a.png", "segments_info": [{"id": 5, "category_id": 1, "area": 24,
                                                                      "iscrowd": 0}]}
    (tmp_path / "gt").mkdir()
    Image.fromarray(pe.id2rgb(gt_map)).save(tmp_path / "gt" / "a.png")
    (tmp_path / "gt.json").write_text(json.dumps({"categories": cats, "annotations": [gt_ann]}))
    ev = pe.PanopticEvaluator(str(tmp_path / "gt.json"), str(tmp_path / "gt"), output_dir=str(tmp_path / "out"))
    pm = np.full((4, 6), 3, np.int32)
    segs = {"unlisted": [], "category": [{"id": 3, "category_id": 4}],
            "missing": [{"id": 3, "category_id": 1}, {"id": 9, "category_id": 1}],
            "no_prediction": [{"id": 3, "category_id": 1}], "size": [{"id": 3, "category_id": 1}]}[case]
    if case == "size":
        pm = pm[:, :-1]
    pred = {"image_id": 8 if case == "no_prediction" else 7, "file_name": "a.png", "segments_info": segs,
            "png_string": pe.png_of(pm), "label_map": torch.from_numpy(pm).to(DEV)}
    if case == "size":
        with pytest.raises(ValueError):
            ev.update([pred])
    else:
        ev.update([pred])
        with pytest.raises(KeyError if case != "no_prediction" else Exception):
            ev.summarize()
    torch.cuda.synchronize()
