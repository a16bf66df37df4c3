"""MultiSequenceTracker with segmentation masks and attention maps on the CPU suite.

The batched decision entry is substituted by its host build (as in test_multi_tracker_cpu.py), the mask head and the
resolution take their host routes.  A masked `Mux` steps the six reference-recorded MOTS cases as sequences of one run
(some joining late); each must reproduce its fixture exactly.  The vanilla attention-map model runs through
`GraphedDetector.batched` without graphs; each sequence must reproduce the recorded maps.  Also: the ragged
`batched_mask_logits` against single calls, the batched helpers against the single ones, and the argument checks of
the two batched C entries."""
import ctypes
import os

import numpy as np
import pytest
import torch

import attention_map_fixtures as amf
import detr_fixtures as df
import multi_tracker_fixtures as mtf
import track_mask_fixtures as tmf
import tracker_fixtures as tf
from conftest import load_golden
from test_attention_maps_cpu import check_against_golden
from test_multi_tracker_cpu import _oracle_msda, host_multi, host_single, libs  # noqa: F401  (fixtures)
from test_track_masks_cpu import check_masks_against_gold
from trackformer_b200.deformable_detr import DeformablePostProcess, PostProcess
from trackformer_b200.mots import encode, label_map_rle, label_maps_rle, write_results
from trackformer_b200.multi_tracker import MultiSequenceTracker
from trackformer_b200.segmentation import PostProcessSegm, resolve_track_masks, resolve_track_masks_many

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


class MaskedMux(mtf.Mux):
    """`Mux` over MaskedScriptedDetectors: `batched_mask_logits` hands back each image's scripted mask rows, indexed by
    the real rows the decision kernel reports, as `GraphedDetector.batched_mask_logits` does."""
    has_mask_head = True

    def batched(self, samples, targets, prev_features):
        dets, seen = self.dets, {}
        self.dets = [lambda *a, i=i: seen.setdefault(i, dets[i](*a)) for i in range(len(dets))]
        try:
            res = super().batched(samples, targets, prev_features)
        finally:
            self.dets = dets
        images = samples[:, 0, 0, 0].long().tolist()
        self.last_batched = ([seen[i][0]["pred_masks"][0] for i in images], res[2])
        return res

    def batched_mask_logits(self, src_rows, sizes, call=None):
        masks, _ = self.last_batched if call is None else call
        rows, picked, o = [int(r) for r in src_rows], [], 0
        for b, n in enumerate(sizes):
            picked += [masks[b][r] for r in rows[o:o + n]]
            o += n
        return torch.stack(picked) if picked else torch.zeros((0,) + tmf.MASK_HW)


class _View:
    """The shared detector as one sequence sees it: its own `overflow_boxes` (the cases differ in it)."""

    def __init__(self, det, overflow):
        self._det, self.overflow_boxes = det, overflow

    def __getattr__(self, name):
        return getattr(self._det, name)


def _case_blobs(scene, seq):
    for blob in tmf.blobs(scene):
        blob["img"] = torch.full((1, 3, 8, 8), float(seq))
        yield blob


def _run_cases(host_multi, mask_rle, late=(1, 4), device="cpu", cls=None):  # noqa: F811
    """the six MOTS cases as sequences of one run, those in `late` joining three steps late; returns the sequences'
    trackers, their per-frame ids and their scripted detectors"""
    cases = list(tf.CASES)
    dets = [tmf.MaskedScriptedDetector(tf.Scene(seed=0), overflow_boxes=tf.CASES[c]["overflow"]).to(device)
            for c in cases]
    base = host_multi if cls is None else cls

    class PerCase(base):
        def start(self, key, tracker_cfg=None):
            super().start(key, tf.tracker_cfg(cases[key]))
            self._seqs[key].obj_detector = _View(self.obj_detector, tf.CASES[cases[key]]["overflow"])
    mux = MaskedMux(dets)
    if device != "cpu":
        mux = mux.to(device)
    tr = PerCase(mux, {"bbox": DeformablePostProcess(), "segm": PostProcessSegm()}, tf.BASE_CFG,
                 mask_rle=mask_rle, max_batch=len(cases))
    its = {s: _case_blobs(det.scene, s) for s, det in enumerate(dets)}
    per_frame = {s: [] for s in its}
    for step in range(tf.N_FRAMES + 3):
        batch = {}
        for s, it in its.items():
            if s in late and step < 3:
                continue
            if s not in tr._seqs:
                tr.start(s)
            blob = next(it, None)
            if blob is not None:
                batch[s] = blob
        tr.step(batch)
        for s in batch:
            seq = tr.sequence(s)
            per_frame[s].append([t.id for t in seq.tracks] + [-1] + [t.id for t in seq.inactive_tracks])
    return cases, tr, per_frame, dets


def _summary(seq, per_frame):
    out = tf.summarise(seq)
    width = max(len(p) for p in per_frame)
    out["per_frame_ids"] = np.asarray([p + [-2] * (width - len(p)) for p in per_frame], np.int64)
    out["labels"] = tmf.label_maps(seq, tf.N_FRAMES, (tf.IMG_H, tf.IMG_W))
    return out


def test_masked_sequences_match_reference_fixtures(host_multi):  # noqa: F811
    cases, tr, per_frame, _ = _run_cases(host_multi, mask_rle=False)
    for s, case in enumerate(cases):
        out = _summary(tr.sequence(s), per_frame[s])
        gold = check_masks_against_gold(out, f"tracker_masks_{case}")
        for key in gold.files:
            if key == "rows":       # the box post-processing ran at another batch layout (test_multi_tracker_cpu.py)
                np.testing.assert_allclose(out[key][:, 3:], gold[key][:, 3:], rtol=1e-6, atol=1e-4)
            elif key not in ("labels", "prev_log"):     # prev_log: what the scripted detector was handed, not ours
                np.testing.assert_array_equal(out[key], gold[key], err_msg=f"{case}: {key}")
        assert all(t.mask is not None and t.mask.shape == (tf.IMG_H, tf.IMG_W) for t in tr.sequence(s).tracks)


def test_masked_sequences_rle_write_the_device_tracker_file(host_multi, host_single, tmp_path):  # noqa: F811
    """mask_rle=True: each sequence's MOTS20 result file equals a host DeviceTracker's on that sequence alone"""
    cases, tr, _, _ = _run_cases(host_multi, mask_rle=True)
    for s, case in enumerate(cases):
        scene = tf.Scene(seed=0)
        det = tmf.MaskedScriptedDetector(scene, overflow_boxes=tf.CASES[case]["overflow"])
        ref = host_single(det, {"bbox": DeformablePostProcess(), "segm": PostProcessSegm()}, tf.tracker_cfg(case),
                          False, mask_rle=True)
        for blob in tmf.blobs(scene):
            ref.step(blob)
        got = tr.sequence(s).results
        assert all(isinstance(r["mask"], dict) for fr in got.values() for r in fr.values())
        a = write_results(ref.results, str(tmp_path / "ref"), case)
        b = write_results(got, str(tmp_path / "multi"), case)
        assert open(a, "rb").read() == open(b, "rb").read() and os.path.getsize(a) > 0


def test_orig_size_change_with_stale_masks_raises(host_multi):  # noqa: F811
    scene = tf.Scene()
    det = tmf.MaskedScriptedDetector(scene)
    tr = host_multi(MaskedMux([det]), {"bbox": DeformablePostProcess(), "segm": PostProcessSegm()},
                    tf.tracker_cfg("reid_embedding"))
    tr.start(0)
    with pytest.raises(ValueError, match="orig_size"):
        for t, blob in enumerate(_case_blobs(scene, 0)):
            blob["orig_size"] = torch.tensor([[tf.IMG_H + t, tf.IMG_W]])
            tr.step({0: blob})


def test_attention_maps_of_several_sequences_match_reference(host_multi):  # noqa: F811
    """the vanilla fixture model through GraphedDetector.batched (no graphs), three sequences of the recorded video, one
    joining two steps late: each reproduces the recorded maps"""
    from trackformer_b200.graphed_detector import GraphedDetector
    gold = load_golden("attention_maps", "tracker_")
    model, _ = df.build(True, False, masks=False)
    amf.condition_(model, gold["class_bias"])
    model.tracking()
    cfg = dict(tf.BASE_CFG)
    cfg.update(amf.golden_cfg(gold))
    tr = host_multi(GraphedDetector(model, bucket=3, use_graphs=False), {"bbox": PostProcess()}, cfg,
                    generate_attention_maps=True, max_batch=3)
    assert model.generate_attention_maps
    frames = list(amf.blobs())
    late = {2: 2}
    n_queries = {s: [] for s in range(3)}
    with torch.no_grad():
        for step in range(len(frames) + 2):
            batch = {}
            for s in range(3):
                t = step - late.get(s, 0)
                if t == 0:
                    tr.start(s)
                if 0 <= t < len(frames):
                    seq = tr.sequence(s)
                    n_queries[s].append(len(seq.tracks) + len(seq.inactive_tracks))
                    batch[s] = frames[t]
            tr.step(batch)
    for s in range(3):
        res = amf.summarise(tr.sequence(s))
        check_against_golden(res, gold)
        np.testing.assert_array_equal(n_queries[s], gold["n_queries"])
        assert all(t.attention_map is not None for t in tr.sequence(s).tracks)


def test_constructor_accepts_what_it_batches():
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args
    model = build_model(default_args(tracking=True, device="cpu", enc_layers=1, dec_layers=1, masks=True))[0]
    posts = {"bbox": DeformablePostProcess(), "segm": PostProcessSegm()}
    assert isinstance(MultiSequenceTracker(model, posts, tf.BASE_CFG).obj_detector, GraphedDetector)
    box_only = build_model(default_args(tracking=True, device="cpu", enc_layers=1, dec_layers=1))[0]
    with pytest.raises(ValueError, match="masks"):
        MultiSequenceTracker(box_only, posts, tf.BASE_CFG)
    with pytest.raises(ValueError, match="attention maps"):                  # a deformable decoder
        MultiSequenceTracker(model, posts, tf.BASE_CFG, generate_attention_maps=True)
    vanilla, _ = df.build(True, False, masks=True)
    tr = MultiSequenceTracker(vanilla, posts, tf.BASE_CFG, generate_attention_maps=True)
    assert vanilla.generate_attention_maps and tr.masks
    MultiSequenceTracker(vanilla, {"bbox": PostProcess()}, tf.BASE_CFG)
    assert not vanilla.generate_attention_maps


def distinct_masks_(model):
    """Make the mask head's logits depend on the query.  With canonical weights the per-image terms (the lay1 input
    map and the FPN adapters) swamp the attention-map channels, so every query row of an image gets the same mask to
    ~1e-7.  Sharpen the attention, amplify its lay1 channels and drop the adapters: rows of one image then differ by
    far more than batch noise, so a track given another row's mask, or pixels going to the wrong one of two
    overlapping tracks, show."""
    mh = model.mask_head
    with torch.no_grad():
        model.bbox_attention.q_linear.weight.mul_(3.0)
        mh.lay1.weight[:, model.hidden_dim:].mul_(1000.0)
        for adapter in (mh.adapter1, mh.adapter2, mh.adapter3):
            adapter.weight.zero_()
            adapter.bias.zero_()
    return model


def min_row_spread(x):
    """the smallest max-abs difference between two rows of x [P, h, w]"""
    flat = x.flatten(1)
    return min(float((flat[i] - flat[j]).abs().max()) for i in range(len(flat)) for j in range(i + 1, len(flat)))


def test_batched_mask_logits_equal_single_calls(monkeypatch):
    """the ragged head over a different set of real rows per image (one image without any) equals each image's rows
    through batch-1 GraphedDetector.mask_logits; the rows differ by far more than the tolerance, so a row shifted by
    one would fail"""
    from test_model_parity_cpu import build
    import model_fixtures as mf
    from trackformer_b200.graphed_detector import GraphedDetector
    _oracle_msda(monkeypatch)
    model, _ = build(True, False, masks=True)
    mf.canonical_weights_(model, 0)
    distinct_masks_(model)
    model.tracking()
    g = torch.Generator().manual_seed(3)
    imgs = torch.randn(3, 3, 64, 96, generator=g)
    ks, nq = [5, 0, 11], model.num_queries
    targets = [None if k == 0 else {"track_query_boxes": torch.rand(k, 4, generator=g) * 0.5 + 0.2,
                                    "track_query_hs_embeds": torch.randn(k, model.hidden_dim, generator=g)}
               for k in ks]
    rows = [[0, 4, 5 + nq - 1], [], [10, 3, 11, 11 + nq - 1]]
    det = GraphedDetector(model, bucket=8, use_graphs=False)
    with torch.no_grad():
        det.batched(imgs, targets)
        call = det.last_batched
        got = det.batched_mask_logits([r for rs in rows for r in rs], [len(r) for r in rows])
        alone = det.batched_mask_logits(rows[2], [0, 0, len(rows[2])], call)
        assert got.shape == (7,) + got.shape[-2:] and alone.shape[0] == 4
        tol = 1e-6
        spread = min_row_spread(got)
        assert spread > 100 * tol, spread
        torch.testing.assert_close(alone, got[3:], rtol=0, atol=tol)
        o = 0
        for b, k in enumerate(ks):
            det(imgs[b:b + 1], None if k == 0 else [targets[b]])
            if rows[b]:
                want = det.mask_logits(rows[b])[0]
                torch.testing.assert_close(got[o:o + len(rows[b])], want, rtol=0, atol=tol)
                shifted = det.mask_logits([r - 1 if r else 1 for r in rows[b]])[0]     # what an off-by-one gives
                assert float((got[o:o + len(rows[b])] - shifted).abs().max()) > 100 * tol
            o += len(rows[b])
        with pytest.raises(ValueError):
            det.batched_mask_logits([0], [1, 0], call)


def test_batched_helpers_equal_single_ones_on_the_host():
    rng = np.random.default_rng(4)
    labels = [rng.integers(-2, 5, (13, 9)).astype(np.int32), rng.integers(-1, 3, (7, 21)).astype(np.int32)]
    ids = [[0, 3, 9], []]
    assert label_maps_rle([torch.from_numpy(lab) for lab in labels], ids) == [label_map_rle(labels[0], ids[0]), []]
    assert label_maps_rle(labels, ids)[0] == [encode(labels[0] == i) for i in ids[0]]
    with pytest.raises(ValueError):
        label_maps_rle(labels, [[1], [-1]])
    jobs = []
    for h, w, orig in ((5, 7, (19, 27)), (6, 4, (11, 9))):
        logits = torch.from_numpy(rng.normal(0, 4, (3, h, w)).astype(np.float32))
        jobs.append((logits, [2, 0], [7, 4], None, (4 * h, 4 * w), (4 * h - 1, 4 * w), orig))
    many = resolve_track_masks_many(jobs)
    assert len(many) == 2 and all(torch.equal(m, resolve_track_masks(*j)) for m, j in zip(many, jobs))
    assert resolve_track_masks_many([]) == []


# ---------------------------------------------------------------------------------------------- C-entry arguments
class _MasksArgs(ctypes.Structure):
    """TfbTrackMasksArgs (include/tfb200_fused.h)"""
    _fields_ = ([(n, ctypes.c_void_p) for n in ("logits", "src", "ids", "prev_label", "label")]
                + [(n, ctypes.c_int) for n in ("T", "h", "w", "size_h", "size_w", "crop_h", "crop_w", "H", "W")])


class _RleMap(ctypes.Structure):
    """TfbMaskRleMap (include/tfb200_fused.h)"""
    _fields_ = [("label", ctypes.c_void_p), ("ids", ctypes.c_void_p), ("H", ctypes.c_int), ("W", ctypes.c_int),
                ("T", ctypes.c_int)]


@pytest.fixture(scope="module")
def lib():
    from trackformer_b200 import _build
    return ctypes.CDLL(_build.build_library())


def test_track_masks_batched_entry_rejects_bad_arguments(lib):
    """-1 NULL pointer, -2 bad n or shape, 0 when no image has tracks; nothing touches a device"""
    f = lib.tfb200_track_masks_batched_f32
    f.restype, f.argtypes = ctypes.c_int, [ctypes.POINTER(_MasksArgs), ctypes.c_int, ctypes.c_void_p]
    one = lib.tfb200_track_masks_f32
    one.restype = ctypes.c_int
    one.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_int] * 9 + [ctypes.c_void_p]
    good = _MasksArgs(16, 16, 16, None, 16, 1, 8, 8, 30, 30, 30, 30, 60, 60)
    args = (_MasksArgs * 17)(*([good] * 17))
    assert f(None, 1, None) == -1
    assert f(args, 0, None) == -2 and f(args, 17, None) == -2 and f(args, -3, None) == -2
    bads = []
    for name, value in (("src", None), ("ids", None), ("label", None), ("T", -1), ("h", 0), ("crop_h", 31),
                        ("H", 0), ("W", -5), ("T", (1 << 24) + 1)):
        bad = _MasksArgs.from_buffer_copy(good)
        setattr(bad, name, value)
        bads.append(bad)
    for bad in bads:
        want = one(bad.logits, bad.src, bad.ids, bad.prev_label, bad.label, bad.T, bad.h, bad.w, bad.size_h,
                   bad.size_w, bad.crop_h, bad.crop_w, bad.H, bad.W, None)
        assert want < 0
        for pos in (0, 7, 15):
            a = (_MasksArgs * 16)(*([good] * 16))
            a[pos] = bad
            assert f(a, 16, None) == want
    empty = _MasksArgs.from_buffer_copy(good)
    empty.T = 0
    assert f((_MasksArgs * 16)(*([empty] * 16)), 16, None) == 0


def _layout_bytes(shapes):
    """The encoder's workspace: per region (hash keys and values, per-track words, chunk counts, column-major track
    indices, boundary lists) the maps' parts back to back, each region 256-byte aligned.  For one map this is the
    single-map layout the encoder has always had."""
    def align(v):
        return (v + 255) // 256 * 256
    S = T = N = counts = 0
    for h, w, t in shapes:
        slots = 64
        while slots < 2 * t:
            slots *= 2
        S, T, N = S + slots, T + t, N + h * w
        counts += t * -(-(h * w) // 2048)
    return (2 * align(4 * S) + 3 * align(4 * T) + align(8 * T) + align(4 * counts) + align(4 * N)
            + align(8 * N))


def test_mask_rle_batched_entry_rejects_bad_arguments(lib):
    """-1 NULL pointer, -2 bad n, shape, short workspace or the int32 boundary-offset bound (sum of 2 H W < 2^31),
    0 when no map has tracks; the size queries agree with the single ones for one map and return 0 past the bound"""
    vp = ctypes.c_void_p
    ws = lib.tfb200_mask_rle_batched_workspace_bytes
    ws.restype, ws.argtypes = ctypes.c_size_t, [ctypes.POINTER(_RleMap), ctypes.c_int]
    mx = lib.tfb200_mask_rle_batched_max_bytes
    mx.restype, mx.argtypes = ctypes.c_int64, [ctypes.POINTER(_RleMap), ctypes.c_int]
    ws1 = lib.tfb200_mask_rle_workspace_bytes
    ws1.restype, ws1.argtypes = ctypes.c_size_t, [ctypes.c_int] * 3
    mx1 = lib.tfb200_mask_rle_max_bytes
    mx1.restype, mx1.argtypes = ctypes.c_int64, [ctypes.c_int] * 3
    f = lib.tfb200_mask_rle_batched_i32
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.POINTER(_RleMap), ctypes.c_int, vp, ctypes.c_size_t, vp, vp, ctypes.c_int64, vp]

    def maps(*shapes):
        return (_RleMap * len(shapes))(*[_RleMap(16, 16, h, w, t) for h, w, t in shapes])
    for h, w, t in ((8, 8, 1), (1080, 1920, 100), (3, 4, 0), (480, 640, 7), (2049, 1, 3)):
        assert ws1(h, w, t) == _layout_bytes([(h, w, t)]), (h, w, t)
        assert ws(maps((h, w, t)), 1) == ws1(h, w, t) and mx(maps((h, w, t)), 1) == (mx1(h, w, t) if t else 0)
    two = maps((1080, 1920, 40), (480, 640, 9))
    assert mx(two, 2) == mx1(1080, 1920, 40) + mx1(480, 640, 9)
    assert ws(two, 2) == _layout_bytes([(1080, 1920, 40), (480, 640, 9)])
    # the bound: 16 maps of 2^26 pixels hold 2^31 boundaries; 15 do not
    assert ws(maps(*[(8192, 8192, 1)] * 15), 15) > 0 and mx(maps(*[(8192, 8192, 1)] * 15), 15) > 0
    big = maps(*[(8192, 8192, 1)] * 16)
    assert ws(big, 16) == 0 and mx(big, 16) == 0
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, vp)
    assert f(big, 16, p, 1 << 40, p, p, 100, None) == -2
    small = maps((8, 8, 2), (8, 8, 3))
    need = ws(small, 2)
    assert f(None, 2, p, need, p, p, 100, None) == -1
    assert f(small, 2, None, need, p, p, 100, None) == -1
    assert f(small, 2, p, need, None, p, 100, None) == -1
    assert f(small, 2, p, need, p, None, 100, None) == -1
    for n in (0, 17, -1):
        assert f(maps(*[(8, 8, 1)] * 17), n, p, need, p, p, 100, None) == -2
    for pos, name, value, rc in ((1, "label", None, -1), (0, "ids", None, -1), (1, "H", 0, -2), (0, "W", -1, -2),
                                 (1, "T", -1, -2), (0, "T", (1 << 24) + 1, -2)):
        bad = maps((8, 8, 2), (8, 8, 3))
        setattr(bad[pos], name, value)
        assert f(bad, 2, p, need, p, p, 100, None) == rc, name
    assert f(maps((1 << 15, 1 << 14, 1)), 1, p, need, p, p, 100, None) == -2      # H * W > 2^28
    assert f(small, 2, p, need, p, p, -1, None) == -2                            # capacity
    assert f(small, 2, p, need - 1, p, p, 100, None) == -2                       # workspace too small
    assert f(maps((8, 8, 0), (9, 9, 0)), 2, p, 0, p, p, 0, None) == 0
