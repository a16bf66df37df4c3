"""Attention maps of the vanilla-DETR tracker on the CPU: Tracker(generate_attention_maps=True) over DETRSegmTracking
against the reference's own tracker (tests/golden/make_golden_attention_maps.py), the maps of box-only DETRTracking
against the stock last-layer cross-attention, the switch left off, the refused detectors and the C entry's argument
checks."""
import ctypes

import numpy as np
import pytest
import torch

import attention_map_fixtures as amf
import detr_fixtures as df
import tracker_fixtures as tf
from conftest import load_golden


def _build(tracking, multi_frame, **kw):
    return df.build(tracking, multi_frame, **kw)


def check_against_golden(res, gold, map_atol=1e-5):
    for key in ("num_reids", "track_num", "active_ids", "inactive_ids"):
        np.testing.assert_array_equal(res[key], gold[key], err_msg=key)
    np.testing.assert_array_equal(res["rows"][:, :3], gold["rows"][:, :3])
    np.testing.assert_allclose(res["rows"], gold["rows"], rtol=1e-4, atol=1e-3)
    np.testing.assert_array_equal(res["map_keys"], gold["map_keys"])
    assert res["maps"].dtype == np.float32 and res["maps"].shape == gold["maps"].shape
    np.testing.assert_allclose(res["maps"], gold["maps"], rtol=1e-4, atol=map_atol)


@pytest.mark.parametrize("name,segm", [("attention_maps", False), ("attention_maps_segm", True)])
def test_tracker_reproduces_reference_maps(name, segm):
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.segmentation import PostProcessSegm
    from trackformer_b200.tracker import Tracker
    gold = load_golden(name, "tracker_")
    assert gold["maps"].shape[1:] == (8, 10) and int(gold["num_reids"]) > 0 and len(set(gold["map_keys"][:, 0])) > 1
    # tracks kept through their own track queries, tracks inactive for a frame or more that come back through theirs,
    # tracks still inactive at the end, and track-query counts that cross the buckets of 3 of the GPU test's replay
    assert all(amf.events(gold).values()) and len(gold["inactive_ids"]) > 0
    if segm:                    # masks enter no decision: the same rows and maps as with the box post-processing alone
        box = load_golden("attention_maps", "tracker_")
        for key in ("rows", "map_keys", "maps", "n_queries"):
            np.testing.assert_array_equal(gold[key], box[key])
    posts = {"bbox": PostProcess()}
    if segm:
        posts["segm"] = PostProcessSegm()
    res = amf.run_sequence(_build, Tracker, posts, amf.golden_cfg(gold), gold["class_bias"])
    check_against_golden(res, gold)
    np.testing.assert_array_equal(res["n_queries"], gold["n_queries"])
    # every result row carries a map: [h, w] float32 summing to 1 over the unpadded frame
    np.testing.assert_allclose(res["maps"].sum((1, 2)), 1.0, rtol=0, atol=1e-5)
    assert len(res["map_keys"]) == len(res["rows"])


def test_box_only_maps_equal_the_stock_cross_attention():
    """DETRTracking (no mask head; the reference's hook fails there): each result map is the row of the stock last
    decoder layer's multihead_attn(need_weights=True) weights that the track took this frame."""
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.tracker import Tracker
    gold = load_golden("attention_maps", "tracker_")
    tracker, model = amf.build_tracker(_build, Tracker, {"bbox": PostProcess()}, amf.golden_cfg(gold),
                                       gold["class_bias"], masks=False)
    assert type(model).__name__ == "DETRTracking" and model.generate_attention_maps
    seen = []
    hook = model.transformer.decoder.layers[-1].multihead_attn.register_forward_hook(
        lambda mod, inp, out: seen.append(out[1]))
    checked = 0
    try:
        with torch.no_grad():
            for blob in amf.blobs():
                seen.clear()
                tracker.step(blob)
                assert len(seen) == 1 and seen[0] is not None
                stock = seen[0][0]                                        # [Q, h * w]
                h, w = (s // 32 for s in amf.SIZE)
                for k, t in enumerate(tracker.tracks):
                    row = int(tracker._result_rows[k])
                    got = tracker.results[t.id][tracker.frame_index - 1]["attention_map"]
                    assert got.shape == (h, w) and got.dtype == np.float32
                    assert torch.equal(t.attention_map, torch.from_numpy(got))
                    if row >= 0:
                        np.testing.assert_array_equal(got, stock[row].view(h, w).numpy())
                        checked += 1
    finally:
        hook.remove()
    assert checked > 0
    assert all(t.attention_map is None for t in tracker.inactive_tracks)


def test_track_that_is_not_kept_keeps_its_previous_map():
    """steps_termination=2: an active track that misses the track threshold once stays active without a new row and
    keeps the map it had (reference tracker.py:354 only replaces a kept track's map)."""
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.tracker import Tracker
    gold = load_golden("attention_maps", "tracker_")
    cfg = dict(amf.golden_cfg(gold), steps_termination=2)
    tracker, _ = amf.build_tracker(_build, Tracker, {"bbox": PostProcess()}, cfg, gold["class_bias"], masks=False)
    stale = from_track_query = 0
    with torch.no_grad():
        for blob in amf.blobs():
            n_queries = len(tracker.tracks) + len(tracker.inactive_tracks)
            tracker.step(blob)
            f = tracker.frame_index - 1
            for k, t in enumerate(tracker.tracks):
                row = int(tracker._result_rows[k])
                from_track_query += 0 <= row < n_queries
                if row < 0:
                    stale += 1
                    np.testing.assert_array_equal(tracker.results[t.id][f]["attention_map"],
                                                  tracker.results[t.id][f - 1]["attention_map"])
    assert stale > 0 and from_track_query > 0


def test_switch_follows_the_latest_tracker():
    """A Tracker built without maps switches off what an earlier Tracker switched on for the same detector."""
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.tracker import Tracker
    model, _ = df.build(True, False)
    Tracker(model, {"bbox": PostProcess()}, dict(tf.BASE_CFG), True)
    assert model.generate_attention_maps
    Tracker(model, {"bbox": PostProcess()}, dict(tf.BASE_CFG), False)
    assert not model.generate_attention_maps


def test_switch_off_adds_nothing():
    model, _ = df.build(True, False, masks=True)
    model.tracking()
    img = next(amf.blobs((64, 96), 1))["img"]
    with torch.no_grad():
        out = model.detect(img)[0]
        assert "attention_maps" not in out
        model.generate_attention_maps = True
        on = model.detect(img)[0]
    assert on["attention_maps"].shape == (1, model.num_queries, 2, 3)
    assert set(on) == set(out) | {"attention_maps"}
    for key in ("pred_logits", "pred_boxes", "hs_embed"):         # the stock module's need_weights path differs in
        torch.testing.assert_close(on[key], out[key])              # its summation order only
    src = torch.randn(1, model.hidden_dim, 2, 3)
    mask = torch.zeros(1, 2, 3, dtype=torch.bool)
    pos = torch.randn(1, model.hidden_dim, 2, 3)
    qe = torch.randn(5, 1, model.hidden_dim)
    with torch.no_grad():
        assert len(model.transformer(src, mask, qe, pos)) == 3
        assert len(model.transformer(src, mask, qe, pos, need_weights=True)) == 4


def test_tracker_without_the_switch_writes_no_maps():
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.tracker import Tracker
    gold = load_golden("attention_maps", "tracker_")
    model, _ = df.build(True, False)
    amf.condition_(model, gold["class_bias"])
    model.tracking()
    tracker = Tracker(model, {"bbox": PostProcess()}, dict(tf.BASE_CFG, **amf.golden_cfg(gold)), False)
    with torch.no_grad():
        for blob in amf.blobs(n_frames=2):
            tracker.step(blob)
    assert not model.generate_attention_maps and tracker.results
    assert all("attention_map" not in e for r in tracker.results.values() for e in r.values())
    assert all(t.attention_map is None for t in tracker.tracks)


def test_refused_for_deformable_and_scripted_detectors():
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.tracker import Tracker
    scene = tf.Scene()
    with pytest.raises(ValueError):
        Tracker(tf.ScriptedDetector(scene), {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), True)
    model = build_model(default_args(tracking=True, device="cpu", enc_layers=1, dec_layers=1))[0]
    with pytest.raises(ValueError, match="not possible for deformable DETR"):
        Tracker(model, {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), True)


def test_weights_entry_rejects_bad_arguments_without_gpu():
    from trackformer_b200 import _build
    lib = ctypes.CDLL(_build.build_library())
    f = lib.tfb200_dense_attn_weights_f32
    f.restype = ctypes.c_int
    vp, i, fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    f.argtypes = [vp] * 5 + [i] * 4 + [vp, fl, vp]
    buf = ctypes.create_string_buffer(256)
    base = (ctypes.addressof(buf) + 15) & ~15
    p = ctypes.c_void_p(base)
    strides = (ctypes.c_int64 * 4)(512, 256, 512, 256)
    s = ctypes.cast(strides, vp)
    assert f(None, p, None, p, p, 2, 8, 4, 4, s, 0.17, None) == -1      # NULL q
    assert f(p, None, None, p, p, 2, 8, 4, 4, s, 0.17, None) == -1      # NULL k
    assert f(p, p, None, None, p, 2, 8, 4, 4, s, 0.17, None) == -1      # NULL lse
    assert f(p, p, None, p, None, 2, 8, 4, 4, s, 0.17, None) == -1      # NULL weights
    assert f(p, p, None, p, p, 2, 8, 4, 4, None, 0.17, None) == -1      # NULL strides
    assert f(p, p, None, p, p, 0, 8, 4, 4, s, 0.17, None) == -2         # B = 0
    assert f(p, p, None, p, p, 2, 8, 0, 4, s, 0.17, None) == -2         # Lq = 0
    assert f(p, p, None, p, p, 2, 8, 4, 0, s, 0.17, None) == -2         # Lk = 0
    odd = ctypes.c_void_p(base + 4)
    assert f(odd, p, None, p, p, 2, 8, 4, 4, s, 0.17, None) == -2       # q not 16-byte aligned
    strides[2] = 514
    assert f(p, p, None, p, p, 2, 8, 4, 4, s, 0.17, None) == -2         # k rows not 16-byte aligned
    strides[2], strides[1] = 512, 258
    assert f(p, p, None, p, p, 2, 8, 4, 4, s, 0.17, None) == -2         # q batch stride not a multiple of 4


def test_cpu_attention_returns_the_stock_weights():
    from trackformer_b200 import dense_attention
    torch.manual_seed(0)
    mha = torch.nn.MultiheadAttention(256, 8, dropout=0.1).eval()
    q, mem = torch.randn(7, 2, 256), torch.randn(11, 2, 256)
    pad = torch.zeros(2, 11, dtype=torch.bool)
    pad[1, 6:] = True
    out, w = dense_attention.attention(mha, q, mem, mem, pad, need_weights=True)
    want_out, want_w = mha(q, mem, mem, key_padding_mask=pad, need_weights=True)
    torch.testing.assert_close(out, want_out)
    torch.testing.assert_close(w, want_w)
    assert w.shape == (2, 7, 11) and float(w[1, :, 6:].abs().max()) == 0.0
