"""The four evaluators checked against each other and against their own invariances, on the CPU suite.

Each evaluator's tests compare it with a numpy oracle written from the same reading of pycocotools, motmetrics or
panopticapi, so a misreading shared by the two would go unseen.  Here the references are independent:
  * COCO box AP and mask AP of the same rectangles (integer boxes, masks [x1, x2) x [y1, y2), area = w h) are
    bit-identical: the box path (bbIou on float32 widths) and the mask path (RLE decode, bit planes, popcounts) must
    agree on every IoU, crowd union and detection area;
  * MOT on boxes and MOTS on the rectangles' RLEs count the same matches, switches, misses, false positives,
    fragmentations, MT / PT / ML and IDTP, with sums of distances equal to float32 rounding;
  * the MOTS ignore rule equals a dense numpy restatement, and removing a hypothesis by the rule equals leaving it out;
  * every evaluator gives bit-identical results under relabelled ids, permuted detections / tracks / segments,
    another update order or batching, per-sequence or joint evaluation, translation, and a second run.
The scenes are tests/eval_consistency_fixtures.py's.  Here the relations run through the g++ host builds of the
kernels' sources, driven by the product's own host code; tests/test_eval_consistency_gpu.py runs them through the
public CUDA entry points.  The checks are the `check_*` functions, written against a backend that evaluates."""
import ctypes
import json
import os

import numpy as np
import pytest

import eval_consistency_fixtures as ef
import host_twin
import mot_eval_fixtures as mf
from test_coco_eval_cpu import host_eval
from test_mot_eval_cpu import host_counters as mot_host_counters
from test_mots_eval_cpu import host_counters as mots_host_counters
from trackformer_b200 import mot_eval, mots_eval
from trackformer_b200 import panoptic_eval as pe

MOT_COUNTS = {"matches": mot_eval._MATCH, "switches": mot_eval._SWITCH, "misses": mot_eval._MISS,
              "fp": mot_eval._FP, "frag": mot_eval._FRAG, "mt": mot_eval._MT, "pt": mot_eval._PT,
              "ml": mot_eval._ML, "idtp": mot_eval._IDTP}


def _compile(tmp_path_factory, name, argtypes):
    lib = host_twin.build(f"{name}_host", tmp_path_factory.mktemp(name))
    for fn, (args, res) in argtypes.items():
        getattr(lib, fn).argtypes, getattr(lib, fn).restype = args, res
    return lib


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    """The host builds of coco_eval_core.h, mot_eval_core.h, mots_eval_core.h and panoptic_core.h."""
    vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t
    coco = _compile(tmp_path_factory, "coco_eval", {
        "tfb200_coco_match_host": ([vp, i32, i32, i32, vp, vp, vp, i64, vp, i32] + [vp] * 11
                                   + [i32, vp, i32, i32, i32, i64, i64, i64, i64, vp, vp, vp, vp, vp], i32),
        "tfb200_coco_accumulate_host": ([vp, vp, vp, i64, vp, i32, i64, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp,
                                         vp, vp, vp], i32)})
    mot = _compile(tmp_path_factory, "mot_eval", {
        "tfb200_mot_eval_host_workspace_bytes": ([i32, i32, i64, i64, i64, i32, i32, i64], sz),
        "tfb200_mot_eval_host": ([vp] * 7 + [i32, i32, i64, i64, i64, i32, i32, i64, vp, sz, vp], i32)})
    mots = _compile(tmp_path_factory, "mots_eval", {
        "tfb200_mots_eval_host_workspace_bytes": ([i32, i32, i32, i64, i64, i64, i32, i32, i64, i64, i64], sz),
        "tfb200_mots_eval_host": ([vp] * 9 + [i32, i32, i32, i64, i64, i64, i32, i32, i64, i64, i64, vp, sz, vp],
                                  i32)})
    pq = pe.bind(host_twin.build("panoptic_host", tmp_path_factory.mktemp("panoptic")))
    return {"coco": coco, "mot": mot, "mots": mots, "pq": pq}


class HostBackend:
    """The relations' evaluators: the host builds through the product's packing and summaries."""

    def __init__(self, libs, tmp):
        self.libs, self.tmp = libs, tmp

    def coco(self, dataset, updates, iou_type):
        """(precision, recall, scores, stats) after `update` of each dict in `updates`, in order."""
        return host_eval(self.libs["coco"], dataset, updates, iou_type)

    def mot(self, accums, names):
        """(counters [S, 16], summary DataFrame)"""
        out = mot_host_counters(self.libs["mot"], accums)
        return out, mot_eval.summarize(accums, names, out)[0]

    def mots(self, accums, names):
        """(counters [S, 27], summary DataFrame)"""
        out = mots_host_counters(self.libs["mots"], accums, names)
        return out, mots_eval.summarize(accums, names, out)[0]

    pq_device = "cpu"

    def pq_lib(self):
        return self.libs["pq"]

    def pq_map(self, m):
        return m


@pytest.fixture
def backend(host_lib, tmp_path):
    return HostBackend(host_lib, tmp_path)


def same(a, b):
    """bit-identical tuples / lists of arrays"""
    assert len(a) == len(b)
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape and x.dtype == y.dtype and x.tobytes() == y.tobytes()


# ================================================================ COCO

def check_coco_bbox_equals_segm(backend, dataset, update):
    """Box AP and mask AP of the same rectangles: precision, recall, scores and the 12 stats bit-identical, with
    maxDets 1, 10 and 100 (the M axis), more than 100 detections in one category of one image, crowds and a category
    without GT."""
    assert any(a["iscrowd"] for a in dataset["annotations"])
    assert max(int((p["labels"] == 0).sum()) for p in update.values()) > 100
    gt_cats = {a["category_id"] for a in dataset["annotations"]}
    assert any(c["id"] not in gt_cats for c in dataset["categories"])
    box = backend.coco(dataset, [update], "bbox")
    segm = backend.coco(dataset, [update], "segm")
    same(box, segm)
    p, r, s, stats = box
    assert stats[0] > 0 and (r[:, :, :, 0] == -1).any() and (p[0, :, :, 1:, 2] > 0).any()   # non-trivial
    return box


def check_coco_invariances(backend, dataset, update, iou_type, seed):
    rng = np.random.default_rng(seed)
    base = backend.coco(dataset, [update], iou_type)
    p, r, s, stats = base
    # relabelled categories, annotation ids and image ids: the K axis follows the category ids' sorted order
    ds2, up2, k_of = ef.coco_relabel(dataset, update, rng)
    p2, r2, s2, stats2 = backend.coco(ds2, [up2], iou_type)
    same((p, r, s), (p2[:, :, k_of], r2[:, k_of], s2[:, :, k_of]))
    # the stats average the categories in id order with numpy: another order may move the last bit
    assert np.allclose(stats, stats2, rtol=0, atol=1e-15)
    ds3, up3, k3 = ef.coco_relabel(dataset, update, rng, cats=False)
    assert (k3 == np.arange(len(k3))).all()
    same(base, backend.coco(ds3, [up3], iou_type))
    # detections permuted inside each image
    same(base, backend.coco(dataset, [ef.coco_permute(update, rng)], iou_type))
    # images in another order, split over several updates, and a later duplicate of an image (the first record of an
    # image id is the one kept, as the reference's merge keeps it)
    ids = list(update)
    rng.shuffle(ids)
    parts = [{i: update[i] for i in ids[k::3]} for k in range(3)]
    dup = ids[0]
    other = next(i for i in ids if i != dup)
    hw = update[dup]["masks"].shape[2:]
    junk = dict(update[other], masks=update[other]["masks"][:, :, :1, :1].expand(-1, -1, *hw).contiguous())
    parts.append({dup: junk})
    same(base, backend.coco(dataset, [p_ for p_ in parts if p_], iou_type))
    # a second run in the same process
    same(base, backend.coco(dataset, [update], iou_type))
    return base


def check_coco_translation(backend, dataset, update, iou_type, seed):
    """Every box and mask moved by the same integer offset inside the images: bit-identical."""
    rng = np.random.default_rng(seed)
    base = backend.coco(dataset, [update], iou_type)
    left, top, right, bottom = ef.coco_margin(dataset, update)
    assert min(left, top, right, bottom) >= 2
    for dx, dy in ((int(rng.integers(1, right + 1)), -int(rng.integers(1, top + 1))),
                   (-left, bottom)):
        ds2, up2 = ef.coco_translate(dataset, update, dx, dy)
        same(base, backend.coco(ds2, [up2], iou_type))


@pytest.mark.parametrize("seed", range(3))
def test_coco_bbox_equals_segm(backend, seed):
    check_coco_bbox_equals_segm(backend, *ef.coco_scene(seed))


@pytest.mark.parametrize("iou_type", ["bbox", "segm"])
def test_coco_invariances(backend, iou_type):
    check_coco_invariances(backend, *ef.coco_scene(11), iou_type, 11)


@pytest.mark.parametrize("iou_type", ["bbox", "segm"])
def test_coco_translation(backend, iou_type):
    ds, up = ef.coco_scene(12, images=((200, 200, 16), (488, 488, 120), (64, 64, 32), (72, 72, 32)), pad=4)
    check_coco_translation(backend, ds, up, iou_type, 12)


# ================================================================ MOT and MOTS

def _mot_counts(out):
    return {k: out[:, v].copy() for k, v in MOT_COUNTS.items()}


def check_mot_equals_mots(backend, scenes):
    """MOT on the boxes and MOTS on their rectangles: the same counts; sums of distances to float32 rounding; the
    same MOTA (= MOTSA here), IDF1, IDP, IDR, recall and precision."""
    names = list(scenes)
    assert max(ef.max_objects_per_frame(s) for s in scenes.values()) > mot_eval.MAX_CLEAR_COMPONENT
    mo, ms = backend.mot(ef.mot_accums(scenes), names)
    so, ss = backend.mots(ef.mots_accums(scenes), names)
    a, b = _mot_counts(mo), _mot_counts(so)
    for k in MOT_COUNTS:
        assert (a[k] == b[k]).all(), (k, a[k], b[k])
    assert (a["switches"] > 0).any() and (a["frag"] > 0).any() and (a["fp"] > 0).any() and (a["misses"] > 0).any()
    assert (so[:, 16 + mots_eval._XREMOVED] == 0).all()
    d_mot = mo[:, mot_eval._SUMD].copy().view(np.float64)
    d_mots = so[:, mot_eval._SUMD].copy().view(np.float64)
    tp = a["matches"] + a["switches"]
    assert (np.abs(d_mot - d_mots) <= 1e-6 * np.maximum(tp, 1)).all(), (d_mot, d_mots)
    for col in ("idf1", "idp", "idr", "recall", "precision"):
        assert np.array_equal(ms[col].to_numpy(), ss[col].to_numpy(), equal_nan=True), col
    assert np.allclose(ms["mota"].to_numpy(), ss["motsa"].to_numpy(), rtol=0, atol=1e-12, equal_nan=True)
    for col in ("num_false_positives", "num_misses", "num_switches", "num_fragmentations", "mostly_tracked",
                "partially_tracked", "mostly_lost", "num_unique_objects"):
        assert np.array_equal(ms[col].to_numpy(), ss[col].to_numpy()), col


def _mot_relabel(results, frames, rng):
    tmap = dict(zip(results, (int(v) for v in rng.choice(10 ** 6, len(results), replace=False))))
    gids = sorted({g for fr in frames for g in fr["gt"]})
    gmap = dict(zip(gids, (int(v) for v in rng.choice(np.arange(1, 10 ** 6), len(gids), replace=False))))
    return ({tmap[t]: tr for t, tr in results.items()},
            [{"gt": {gmap[g]: b for g, b in fr["gt"].items()}} for fr in frames])


def _mot_permute(results, rng):
    keys = list(results)
    return {keys[i]: results[keys[i]] for i in rng.permutation(len(keys))}


def check_track_invariances(backend, scenes, seed):
    """MOT and MOTS: relabelled GT / track ids, permuted tracks, per-sequence against joint evaluation (per-sequence
    counters equal, OVERALL the sum of the counts), translation and a second run, all bit-identical."""
    rng = np.random.default_rng(seed)
    names = list(scenes)
    for kind, accums_of, run in (("mot", ef.mot_accums, backend.mot), ("mots", ef.mots_accums, backend.mots)):
        base, summary = run(accums_of(scenes), names)
        variants = {"relabel": {n: ef.relabel_track_scene(s, rng) for n, s in scenes.items()},
                    "permute": {n: ef.permute_tracks(s, rng) for n, s in scenes.items()}}
        moved = {}
        for n, s in scenes.items():
            left, top, right, bottom = ef.track_margin(s)
            moved[n] = ef.translate_track_scene(s, int(rng.integers(-left, right + 1)),
                                                int(rng.integers(-top, bottom + 1)))
        variants["translate"] = moved
        for what, sc in variants.items():
            out, _ = run(accums_of(sc), names)
            assert out.tobytes() == base.tobytes(), (kind, what)
        out, _ = run(accums_of(scenes), names)
        assert out.tobytes() == base.tobytes(), (kind, "repeat")
        for s, n in enumerate(names):
            alone, _ = run(accums_of({n: scenes[n]}), [n])
            assert alone.tobytes() == base[s:s + 1].tobytes(), (kind, n)
        ints = [c for c in summary.columns if summary[c].dtype == np.int64]
        for c in ints:
            assert summary[c]["OVERALL"] == summary[c][names].sum(), (kind, c)


def check_mot_invariances_overlapping(backend, seed):
    """MOT on scenes with overlapping boxes and real assignment problems (mot_eval_fixtures: continuous jitter, so no
    two assignments tie; clumps of 2-6 people): relabelled ids and permuted tracks change nothing."""
    rng = np.random.default_rng(seed)
    seqs = {"walk": mf.scene(seed, n_frames=25), "clumps": mf.clumps(seed, n_frames=6, n_clumps=40)}
    names = list(seqs)
    acc = lambda sq: [mot_eval.get_mot_accum(r, fr) for r, fr in sq.values()]
    base, _ = backend.mot(acc(seqs), names)
    assert (base[:, mot_eval._SWITCH] > 0).all() and base[:, mot_eval._CROWS].max() > 1
    relabelled = {n: _mot_relabel(r, fr, rng) for n, (r, fr) in seqs.items()}
    permuted = {n: (_mot_permute(r, rng), fr) for n, (r, fr) in seqs.items()}
    for sq in (relabelled, permuted):
        out, _ = backend.mot(acc(sq), names)
        assert out.tobytes() == base.tobytes()


def check_mots_ignore_rule(backend, scene):
    """The hypotheses without a candidate that lie more than half inside the ignore union (dense numpy) are the
    ones removed: their number is the counter's, and evaluating without them (and without ignore regions) gives the
    same counts.  Hypotheses exactly half inside are kept: they count as false positives."""
    drop = ef.removed_hypotheses(scene)
    half = ef.exactly_half_inside(scene)
    assert drop and half and not (drop & half)
    names = ["s"]
    out, _ = backend.mots(ef.mots_accums({"s": scene}), names)
    x = out[0, 16:]
    n_hyp = sum(len(tr) for tr in scene["hyps"].values())
    assert x[mots_eval._XREMOVED] == len(drop) and x[mots_eval._XKEPT] == n_hyp - len(drop)
    clean, _ = backend.mots(ef.mots_accums({"s": ef.without(scene, drop)}), names)
    assert out[0, :16].tobytes() == clean[0, :16].tobytes()
    assert x[mots_eval._XGTDETS] == clean[0, 16 + mots_eval._XGTDETS]
    fewer, _ = backend.mots(ef.mots_accums({"s": ef.without(scene, drop | half)}), names)
    assert fewer[0, mot_eval._FP] == out[0, mot_eval._FP] - len(half)


@pytest.mark.parametrize("seed", range(2))
def test_mot_equals_mots(backend, seed):
    check_mot_equals_mots(backend, ef.track_scenes(10 * seed))


def test_track_invariances(backend):
    check_track_invariances(backend, ef.track_scenes(40), 40)


@pytest.mark.parametrize("seed", range(2))
def test_mot_invariances_overlapping_boxes(backend, seed):
    check_mot_invariances_overlapping(backend, seed)


@pytest.mark.parametrize("seed", range(3))
def test_mots_ignore_rule_against_dense_masks(backend, seed):
    check_mots_ignore_rule(backend, ef.track_scene(50 + seed, n_frames=10, ignore=True))


# ================================================================ panoptic

def pq_run(backend, data, tmp, order=None, batch=1000, label_maps=True):
    """`PanopticEvaluator` over `data`: the predictions in `order` (image ids; default the GT's), `batch` per
    `update`; the prediction maps given as device `label_map`s or only as PNGs.  Returns (results, tp, fp, fn, iou)."""
    gt_json, pred_json, gmaps, pmaps = data
    os.makedirs(tmp / "gt", exist_ok=True)
    for a in gt_json["annotations"]:
        (tmp / "gt" / a["file_name"]).write_bytes(pe.png_of(gmaps[a["image_id"]]))
    (tmp / "gt.json").write_text(json.dumps(gt_json))
    ev = pe.PanopticEvaluator(str(tmp / "gt.json"), str(tmp / "gt"), output_dir=str(tmp / "out"),
                              device=backend.pq_device, lib=backend.pq_lib())
    preds = {a["image_id"]: a for a in pred_json["annotations"]}
    order = list(order if order is not None else preds)
    for c in range(0, len(order), batch):
        items = []
        for i in order[c:c + batch]:
            p = dict(preds[i], png_string=pe.png_of(pmaps[i]))
            if label_maps:
                p["label_map"] = backend.pq_map(pmaps[i])
            items.append(p)
        ev.update(items)
    results = ev.summarize()
    raw = ev._scorer.result([a["image_id"] for a in gt_json["annotations"]])
    return (results, *raw)


def same_pq(a, b, cmap=None):
    """results dicts and raw per-category arrays bit-identical (categories renamed by cmap)."""
    ra, rb = a[0], b[0]
    for name in ("All", "Things", "Stuff"):
        assert ra[name] == rb[name], name
    cmap = cmap or {c: c for c in ra["per_class"]}
    assert {cmap[c]: v for c, v in ra["per_class"].items()} == rb["per_class"]
    same(a[1:], b[1:])


def check_pq_invariances(backend, data, tmp, seed):
    rng = np.random.default_rng(seed)
    base = pq_run(backend, data, tmp / "base")
    tp, fp, fn, iou = base[1:]
    assert tp.sum() > 5 and fp.sum() > 0 and fn.sum() > 0 and base[0]["Stuff"]["n"] > 0
    relabelled, cmap = ef.pq_relabel(data, rng)
    same_pq(base, pq_run(backend, relabelled, tmp / "relabel"), cmap)
    same_pq(base, pq_run(backend, ef.pq_permute(data, rng), tmp / "permute"))
    ids = [a["image_id"] for a in data[0]["annotations"]]
    for k, b in enumerate((1, 2, 3)):
        order = [ids[i] for i in rng.permutation(len(ids))]
        same_pq(base, pq_run(backend, data, tmp / f"order{k}", order=order, batch=b, label_maps=k != 1))
    dy, dx = (int(v) for v in rng.integers(-8, 9, 2))
    same_pq(base, pq_run(backend, ef.pq_translate(data, dy, dx), tmp / "translate"))
    same_pq(base, pq_run(backend, data, tmp / "base"))                    # a second run
    return base


def check_pq_compute_batching(backend, data, tmp):
    """`pq_compute` over PNG folders: the batch size does not matter, and it equals the evaluator."""
    gt_json, pred_json, gmaps, pmaps = data
    for side, js, maps in (("gt", gt_json, gmaps), ("pred", pred_json, pmaps)):
        os.makedirs(tmp / side, exist_ok=True)
        for a in js["annotations"]:
            (tmp / side / a["file_name"]).write_bytes(pe.png_of(maps[a["image_id"]]))
        (tmp / f"{side}.json").write_text(json.dumps(js))
    args = [str(tmp / "gt.json"), str(tmp / "pred.json"), str(tmp / "gt"), str(tmp / "pred")]
    one = pe.pq_compute(*args, device=backend.pq_device, batch=1, lib=backend.pq_lib())
    many = pe.pq_compute(*args, device=backend.pq_device, batch=16, lib=backend.pq_lib())
    assert one == many
    assert one == pq_run(backend, data, tmp / "ev")[0]


@pytest.mark.parametrize("seed", range(2))
def test_pq_invariances(backend, tmp_path, seed):
    check_pq_invariances(backend, ef.pq_scene(seed), tmp_path, seed)


def test_pq_compute_batching(backend, tmp_path):
    check_pq_compute_batching(backend, ef.pq_scene(7, n_images=6), tmp_path)
