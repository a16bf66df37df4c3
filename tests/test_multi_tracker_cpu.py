"""MultiSequenceTracker on the CPU suite.

The batched decision entry is substituted by its host build (tests/host_build/track_step_batched_host.cpp: the routine
the kernel's CTA b runs, one sequence after the other), as test_track_step_cpu.py substitutes the single entry.  The
scripted scenes and the real detector (GraphedDetector.batched without graphs) then run through the whole batched path
-- grouping, row offsets into the padded outputs, the shared result buffer and its one read-back, slot refill -- and
every sequence must come out as it does tracked alone."""
import ctypes
import os

import numpy as np
import pytest
import torch

import multi_tracker_fixtures as mtf
import tracker_fixtures as tf
from trackformer_b200.deformable_detr import DeformablePostProcess
from trackformer_b200.device_tracker import DeviceTracker, _ArgsC
from trackformer_b200.multi_tracker import MultiSequenceTracker, track_sequences
from trackformer_b200.tracker import Tracker

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("multi_track")
    single = mtf.build_host(tmp, "track_step_host")
    single.tfb200_track_step_host.argtypes = [ctypes.POINTER(_ArgsC)]
    batched = mtf.build_host(tmp, "track_step_batched_host")
    batched.tfb200_track_step_batched_host.argtypes = [ctypes.POINTER(_ArgsC), ctypes.c_int]
    return single, batched


@pytest.fixture(scope="module")
def host_multi(libs):
    _, batched = libs

    class HostMulti(MultiSequenceTracker):
        launches = 0

        def _launch(self, args, n, tensors):
            assert not any(t.is_cuda for t in tensors)
            assert batched.tfb200_track_step_batched_host(args, n) == 0
            HostMulti.launches += 1
    return HostMulti


@pytest.fixture(scope="module")
def host_single(libs):
    single, _ = libs

    class HostSingle(DeviceTracker):
        def _launch(self, args, tensors):
            assert single.tfb200_track_step_host(ctypes.byref(args)) == 0
    return HostSingle


def _rows(results):
    """the rows tracker_fixtures.summarise makes of a finished sequence's results"""
    return np.asarray([[tid, f, int(r["obj_ind"]), float(r["score"])] + [float(v) for v in r["bbox"]]
                       for tid in sorted(results) for f, r in sorted(results[tid].items())], np.float64).reshape(-1, 8)


def _compare(a, b, exact):
    for key in b:
        if key == "rows" and not exact:
            np.testing.assert_array_equal(a[key][:, :3], b[key][:, :3])
            np.testing.assert_allclose(a[key][:, 3:], b[key][:, 3:], rtol=1e-6, atol=1e-4)
        else:
            np.testing.assert_array_equal(a[key], b[key], err_msg=key)


@pytest.mark.parametrize("n", range(1, 17))
def test_batched_entry_equals_single_calls_bit_for_bit(libs, n):
    """Every batched call of an n-sequence run is replayed as n single calls from the same memory: every byte the step
    writes (both state buffers, next-frame queries, integer scratch, header + result rows) must agree."""
    single, batched = libs
    checked = []

    class Checked(MultiSequenceTracker):
        def _launch(self, args, m, tensors):
            spans = [s for b in range(m) for s in mtf.output_spans(args[b])]
            before = [ctypes.string_at(p, k) for p, k in spans]
            for b in range(m):
                single.tfb200_track_step_host(ctypes.byref(args[b]))
            after_single = [ctypes.string_at(p, k) for p, k in spans]
            for (p, k), data in zip(spans, before):
                ctypes.memmove(p, data, k)
            assert batched.tfb200_track_step_batched_host(args, m) == 0
            assert [ctypes.string_at(p, k) for p, k in spans] == after_single
            checked.append(m)

    specs = mtf.sequence_specs(n)
    dets = [make() for _, make, _, _ in specs]
    tr = Checked(mtf.Mux(dets), {"bbox": DeformablePostProcess()}, tf.BASE_CFG, max_batch=n)
    sequences = {}
    for s, ((cfg, _, frames, public), det) in enumerate(zip(specs, dets)):
        sequences[s] = mtf.blobs(det, s, frames, public)
    # sequences start at different frames: the odd ones join two steps late
    its = {s: iter(b) for s, b in sequences.items()}
    for step in range(tf.N_FRAMES + 2):
        batch = {}
        for s, it in its.items():
            if s % 2 and step < 2:
                continue
            if s not in tr._seqs:
                tr.start(s, specs[s][0])
            blob = next(it, None)
            if blob is not None:
                batch[s] = blob
        tr.step(batch)
    assert max(checked) == n and sum(tr.sequence(s).track_num for s in its) > n


@pytest.mark.parametrize("n", [1, 3, 8, 16])
def test_multi_tracker_equals_per_sequence_trackers(host_multi, host_single, n):
    """scripted and noise scenes of every kind (public detections, ReID greedy / embedding, sim-only), each with its
    own thresholds and length, through `track_sequences` with fewer slots than sequences: the results of each equal
    the host Tracker and the single-call device routine on that sequence alone"""
    specs = mtf.sequence_specs(n + 3)
    dets = [make() for _, make, _, _ in specs]
    cfg_of = {s: specs[s][0] for s in range(len(specs))}

    class PerSeqCfg(host_multi):
        def start(self, key, tracker_cfg=None):
            super().start(key, cfg_of[key])
    tr = PerSeqCfg(mtf.Mux(dets), {"bbox": DeformablePostProcess()}, tf.BASE_CFG, max_batch=n)
    before = host_multi.launches
    sequences = {s: mtf.blobs(det, s, frames, public) for s, ((_, _, frames, public), det)
                 in enumerate(zip(specs, dets))}
    got = track_sequences(tr, sequences)
    assert sorted(got) == list(range(len(specs))) and not tr._seqs
    steps = host_multi.launches - before
    assert (steps < sum(f for _, _, f, _ in specs)) == (n > 1)     # sequences really shared launches
    for s, (cfg, make, frames, public) in enumerate(specs):
        outs = []
        for cls in (Tracker, host_single):
            det = make()
            ref = cls(det, {"bbox": DeformablePostProcess()}, cfg, False)
            for blob in mtf.blobs(det, s, frames, public):
                ref.step(blob)
            outs.append(ref)
        a, b = tf.summarise(outs[0]), tf.summarise(outs[1])
        _compare(a, b, exact=False)
        _compare(b, {"rows": _rows(got[s])}, exact=False)     # the post-processing ran at another batch layout
        assert len(got[s]) > 0


def test_multi_tracker_keeps_per_sequence_state(host_multi, host_single):
    """num_reids, track counters, frame index and active / inactive ids of sequences still running"""
    specs = mtf.sequence_specs(3)
    dets = [make() for _, make, _, _ in specs]
    tr = host_multi(mtf.Mux(dets), {"bbox": DeformablePostProcess()}, tf.BASE_CFG, max_batch=3)
    its = {}
    for s, ((cfg, _, frames, public), det) in enumerate(zip(specs, dets)):
        tr.start(s, cfg)
        its[s] = mtf.blobs(det, s, 10, public)
    for _ in range(10):
        tr.step({s: next(it) for s, it in its.items()})
    for s, (cfg, make, _, public) in enumerate(specs):
        det = make()
        ref = host_single(det, {"bbox": DeformablePostProcess()}, cfg, False)
        for blob in mtf.blobs(det, s, 10, public):
            ref.step(blob)
        _compare(tf.summarise(ref), tf.summarise(tr.sequence(s)), exact=True)
        assert tr.get_results(s) is tr.sequence(s).results


def _oracle_msda(monkeypatch):
    from oracle.torch_ref import msda_core_torch
    import trackformer_b200.msda_module as mm

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    monkeypatch.setattr(mm, "MSDeformAttnFunction", _OracleFn)


def _model(multi_frame):
    import model_fixtures as mf
    from test_model_parity_cpu import build
    model, _ = build(True, multi_frame)
    mf.canonical_weights_(model, 0)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 6.0
    model.tracking()
    return model


@pytest.mark.parametrize("multi_frame", [False, True])
def test_batched_forward_equals_single_calls(monkeypatch, multi_frame):
    """GraphedDetector.batched (no graphs) with a different K_b per image, one image without a previous frame: each
    image's real rows equal that image run alone through __call__ (with prev_features=None where it has none)"""
    from trackformer_b200.graphed_detector import GraphedDetector
    _oracle_msda(monkeypatch)
    model = _model(multi_frame)
    size, nq = (64, 96), model.num_queries
    g = torch.Generator().manual_seed(1)
    imgs = torch.randn(3, 3, *size, generator=g)
    ks = [5, 0, 11]
    targets = [None if k == 0 else {"track_query_boxes": torch.rand(k, 4, generator=g) * 0.5 + 0.2,
                                    "track_query_hs_embeds": torch.randn(k, model.hidden_dim, generator=g)}
               for k in ks]
    det = GraphedDetector(model, bucket=8, use_graphs=False)
    with torch.no_grad():
        _, feats, _, _ = det.batched(torch.randn(3, 3, *size, generator=g))          # the "previous frame"
        prev = [(feats, 0), None, (feats, 2)]
        out, _, got_ks, kb = det.batched(imgs, targets, prev)
        assert got_ks == ks and kb == 16
        for b, k in enumerate(ks):
            single_prev = None if prev[b] is None else [f.tensors[b:b + 1] for f in feats]
            if single_prev is not None:
                from trackformer_b200.util import NestedTensor
                single_prev = [NestedTensor(t, f.mask[b:b + 1]) for t, f in zip(single_prev, feats)]
            ref, _, _, _, _ = det(imgs[b:b + 1], None if k == 0 else [targets[b]], single_prev)
            for name in ("pred_logits", "pred_boxes", "hs_embed"):
                torch.testing.assert_close(out[name][b, kb - k:], ref[name][0], rtol=1e-5, atol=1e-5, msg=name)


def test_prev_valid_false_equals_no_previous_frame(monkeypatch):
    """the model's per-image switch: prev_valid False selects the image's own features exactly"""
    _oracle_msda(monkeypatch)
    model = _model(True)
    g = torch.Generator().manual_seed(2)
    imgs = torch.randn(2, 3, 64, 96, generator=g)
    with torch.no_grad():
        _, _, feats, _, _ = model(torch.randn(2, 3, 64, 96, generator=g))
        out, _, _, _, _ = model(imgs, None, feats, torch.tensor([False, True]))
        ref0, _, _, _, _ = model(imgs[:1])
        from trackformer_b200.util import NestedTensor
        ref1, _, _, _, _ = model(imgs[1:], None, [NestedTensor(f.tensors[1:], f.mask[1:]) for f in feats])
    for name in ("pred_logits", "pred_boxes", "hs_embed"):
        torch.testing.assert_close(out[name][:1], ref0[name], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(out[name][1:], ref1[name], rtol=1e-5, atol=1e-5)


def test_multi_tracker_over_the_real_detector(host_multi, monkeypatch):
    """the small real model, sequences of different lengths at two input sizes, one starting late: each sequence's
    results equal the host Tracker over the same padded detector on that sequence alone"""
    from trackformer_b200.graphed_detector import GraphedDetector
    _oracle_msda(monkeypatch)
    model = _model(True)
    gold = np.load(os.path.join(GOLD, "tracker_model_sequence.npz"))
    cfg = {k: float(v) for k, v in zip(gold["cfg_keys"], gold["cfg_values"])}
    cfg["prev_frame_dist"] = int(cfg["prev_frame_dist"])
    full = dict(tf.BASE_CFG)
    full.update(cfg)
    plan = [((128, 160), 4, 5), ((128, 160), 3, 7), ((96, 128), 5, 11), ((128, 160), 2, 13)]   # size, frames, seed

    def seq_blobs(size, n, seed):
        for frame in tf.model_frames(size, n, seed):
            yield {"img": frame[None], "orig_size": torch.tensor([[size[0] * 4, size[1] * 4]])}

    tr = host_multi(GraphedDetector(model, bucket=8, use_graphs=False), {"bbox": DeformablePostProcess()}, full,
                    max_batch=3)
    with torch.no_grad():
        got = track_sequences(tr, {i: (b for b in seq_blobs(*p)) for i, p in enumerate(plan)})
    for i, (size, n, seed) in enumerate(plan):
        ref = Tracker(GraphedDetector(model, bucket=8, use_graphs=False), {"bbox": DeformablePostProcess()}, full)
        with torch.no_grad():
            for blob in seq_blobs(size, n, seed):
                ref.step(blob)
        a, b = tf.summarise(ref)["rows"], _rows(got[i])
        assert len(a) > 0
        np.testing.assert_array_equal(a[:, :3], b[:, :3])
        np.testing.assert_allclose(a[:, 3:], b[:, 3:], rtol=1e-4, atol=1e-3)


def test_constructor_rejects_what_it_does_not_batch():
    det = mtf.Mux([])
    with pytest.raises(ValueError, match="masks"):
        MultiSequenceTracker(det, {"bbox": DeformablePostProcess(), "segm": object()}, tf.BASE_CFG)
    with pytest.raises(ValueError, match="attention maps"):
        MultiSequenceTracker(det, {"bbox": DeformablePostProcess()}, tf.BASE_CFG, generate_attention_maps=True)
    for bad in (0, 17):
        with pytest.raises(ValueError, match="max_batch"):
            MultiSequenceTracker(det, {"bbox": DeformablePostProcess()}, tf.BASE_CFG, max_batch=bad)
    tr = MultiSequenceTracker(det, {"bbox": DeformablePostProcess()}, tf.BASE_CFG, max_batch=1)
    tr.start("a")
    with pytest.raises(RuntimeError, match="running"):
        tr.start("b")
    with pytest.raises(KeyError):
        tr.step({"b": {}})


def test_product_class_refuses_cpu_tensors():
    specs = mtf.sequence_specs(1)
    det = specs[0][1]()
    tr = MultiSequenceTracker(mtf.Mux([det]), {"bbox": DeformablePostProcess()}, specs[0][0])
    tr.start(0)
    with pytest.raises(RuntimeError, match="CUDA"):
        tr.step({0: next(mtf.blobs(det, 0, 1, specs[0][3]))})


def test_batched_entry_argument_checks():
    """n outside 1..16 or an invalid args[b] returns the single entry's error code; nothing is launched (no device
    is touched, so this runs without one)"""
    from trackformer_b200 import _build
    lib = ctypes.CDLL(_build.build_library())
    f = lib.tfb200_track_step_batched_f32
    f.argtypes, f.restype = [ctypes.POINTER(_ArgsC), ctypes.c_int, ctypes.c_void_p], ctypes.c_int
    one = lib.tfb200_track_step_f32
    one.argtypes, one.restype = [ctypes.POINTER(_ArgsC), ctypes.c_void_p], ctypes.c_int
    assert f(None, 1, None) == -1
    good = _ArgsC()
    for name in ("rows", "hs_embeds", "q_boxes", "q_embeds", "result", "iscratch", "fscratch", "dscratch"):
        setattr(good, name, 16)
    for st in (good.inp, good.out):
        for name, _ in st._fields_:
            setattr(st, name, 16)
    good.capacity, good.hidden, good.nq = 256, 8, 4
    args = (_ArgsC * 17)(*([good] * 17))
    assert f(args, 0, None) == -2 and f(args, 17, None) == -2 and f(args, -1, None) == -2
    bad_ptr, bad_shape = _ArgsC.from_buffer_copy(good), _ArgsC.from_buffer_copy(good)
    bad_ptr.rows = None
    bad_shape.capacity = 4096
    for bad in (bad_ptr, bad_shape):
        for pos in (0, 5, 15):
            args = (_ArgsC * 16)(*([good] * 16))
            args[pos] = bad
            assert f(args, 16, None) == one(ctypes.byref(bad), None) < 0
