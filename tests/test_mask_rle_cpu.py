"""COCO run-length encodings of MOTS masks on CPU: trackformer_b200.mots (encode / decode against hand vectors and a
scalar restatement of pycocotools' definition, label_map_rle's host route, the MOTS20 result writer), Tracker with
mask_rle=True on the scripted mask scenes, and the argument checks of the kernel's C entry point."""
import ctypes

import numpy as np
import pytest
import torch

import track_mask_fixtures as tmf
import tracker_fixtures as tf
from trackformer_b200.deformable_detr import DeformablePostProcess
from trackformer_b200.mots import decode, encode, label_map_rle, write_results
from trackformer_b200.segmentation import PostProcessSegm
from trackformer_b200.tracker import Tracker


def scalar_rle(mask):
    """pycocotools rleEncode + rleToString, one pixel and one character at a time"""
    cnts, prev, run = [], 0, 0
    for v in np.asarray(mask, bool).ravel(order="F"):
        if v != prev:
            cnts.append(run)
            run, prev = 0, v
        run += 1
    cnts.append(run)
    s = bytearray()
    for i, x in enumerate(cnts):
        x = int(x) - (int(cnts[i - 2]) if i > 2 else 0)
        more = True
        while more:
            c = x & 0x1F
            x >>= 5
            more = (x != -1) if (c & 0x10) else (x != 0)
            s.append((c | 0x20 if more else c) + 48)
    return cnts, bytes(s)


def _box(h, w, y0, y1, x0, x1):
    m = np.zeros((h, w), bool)
    m[y0:y1, x0:x1] = True
    return m


@pytest.mark.parametrize("mask,counts,string", [
    (np.zeros((3, 4), bool), [12], b"<"),
    (np.ones((3, 4), bool), [0, 12], b"0<"),
    (_box(4, 5, 1, 3, 1, 4), [5, 2, 2, 2, 2, 2, 5], b"5220003"),
    (_box(2, 2, 0, 1, 0, 1), [0, 1, 3], b"013"),
])
def test_encode_hand_vectors(mask, counts, string):
    assert scalar_rle(mask) == (counts, string)
    assert encode(mask) == {"size": list(mask.shape), "counts": string}
    assert (decode(encode(mask)) == mask).all()


def test_encode_person_sized_box_at_1080p():
    m = _box(1080, 1920, 100, 900, 500, 600)
    cnts, s = scalar_rle(m)
    assert len(cnts) == 201 and cnts[:3] == [540100, 800, 280]
    rle = encode(m)
    assert rle["size"] == [1080, 1920] and rle["counts"] == s and s.startswith(b"T^_`0Pi0h8000")
    assert (decode(rle) == m).all()


def _random_masks():
    rng = np.random.default_rng(0)
    for i in range(60):
        h, w = (int(v) for v in rng.integers(1, 30, 2))
        if i % 10 == 0:
            h = 1
        elif i % 10 == 1:
            w = 1
        kind = i % 4
        if kind == 0:                                     # salt and pepper
            m = rng.random((h, w)) < rng.random()
        elif kind == 1:                                   # a run through the bottom of one column and the next's top
            m = np.zeros((h, w), bool)
            x = int(rng.integers(0, w))
            m[h // 2:, x] = True
            if x + 1 < w:
                m[:h // 2 + 1, x + 1] = True
        elif kind == 2:                                   # first and last pixel set
            m = rng.random((h, w)) < 0.3
            m[0, 0] = m[-1, -1] = True
        else:                                             # blocks
            m = np.kron(rng.random((h // 3 + 1, w // 3 + 1)) < 0.5, np.ones((3, 3), bool))[:h, :w]
        yield m


def test_round_trip_and_scalar_definition():
    for m in _random_masks():
        rle = encode(m)
        assert rle["counts"] == scalar_rle(m)[1], m.shape
        back = decode(rle)
        assert back.dtype == bool and back.shape == m.shape and (back == m).all()
    assert encode(np.ones((1, 1), np.uint8))["counts"] == b"01"
    assert (decode({"size": [2, 3], "counts": "6"}) == 0).all()               # str counts decode too


def test_decode_rejects_malformed_strings():
    with pytest.raises(ValueError):
        decode({"size": [3, 4], "counts": b";"})          # 11 pixels for a 3x4 mask
    with pytest.raises(ValueError):
        decode({"size": [3, 4], "counts": b"P"})          # continuation bit on the last character


def test_label_map_rle_host_route():
    rng = np.random.default_rng(1)
    lab = rng.integers(-3, 6, (23, 17)).astype(np.int32)
    lab[:, 4] = 1 << 30
    ids = [2, 9, 0, 1 << 30, 2]                           # absent, repeated and large ids
    got = label_map_rle(torch.from_numpy(lab), ids)
    assert got == [encode(lab == i) for i in ids]
    assert label_map_rle(lab, []) == []
    with pytest.raises(ValueError):
        label_map_rle(lab, [1, -1])


def _results(masks_per_frame, as_rle):
    out = {}
    for f, masks in enumerate(masks_per_frame):
        for tid, m in masks.items():
            out.setdefault(tid, {})[f] = {"mask": encode(m) if as_rle else m, "bbox": np.zeros(4), "score": 1.0}
    return out


def test_write_results_bool_and_rle_give_the_same_file(tmp_path):
    rng = np.random.default_rng(2)
    frames = [{3: rng.random((6, 5)) < 0.4, 0: _box(6, 5, 1, 4, 0, 2)}, {0: np.zeros((6, 5), bool)}]
    a = write_results(_results(frames, False), str(tmp_path / "a"), "MOTS20-02")
    b = write_results(_results(frames, True), str(tmp_path / "b"), "MOTS20-02")
    assert a.endswith("MOTS20-02.txt")
    data = open(a, "rb").read()
    assert data == open(b, "rb").read()
    lines = data.split(b"\r\n")
    assert lines[-1] == b"" and b"\n" not in b"".join(lines)
    want = [(1, 4, frames[0][3]), (1, 1, frames[0][0]), (2, 1, frames[1][0])]     # results' order: track 3, then 0
    for line, (frame, tid, m) in zip(lines[:-1], want):
        assert line == b" ".join([b"%d" % frame, b"%d" % tid, b"2", b"6", b"5", encode(m)["counts"]])


def _run_scripted(cls, case, mask_rle, device="cpu"):
    scene = tf.Scene(seed=0)
    det = tmf.MaskedScriptedDetector(scene, overflow_boxes=tf.CASES[case]["overflow"]).to(device)
    tr = cls(det, {"bbox": DeformablePostProcess(), "segm": PostProcessSegm()}, tf.tracker_cfg(case), False,
             mask_rle=mask_rle)
    tr.reset()
    for blob in tmf.blobs(scene):
        tr.step(blob)
    return tr


def check_rle_results(plain, rle):
    """same results frame by frame; each RLE is the bool mask's encoding; returns the number of masks compared"""
    assert list(plain) == list(rle)
    n = 0
    for tid in plain:
        assert list(plain[tid]) == list(rle[tid])
        for f, a in plain[tid].items():
            b = rle[tid][f]
            assert set(a) == set(b)
            for key in a:
                if key != "mask":
                    np.testing.assert_array_equal(a[key], b[key], err_msg=key)
            assert isinstance(b["mask"], dict) and b["mask"] == encode(a["mask"])
            assert (decode(b["mask"]) == a["mask"]).all()
            n += 1
    return n


@pytest.mark.parametrize("case", list(tf.CASES))
def test_tracker_mask_rle_equals_bool_masks(case, tmp_path):
    plain = _run_scripted(Tracker, case, False)
    rle = _run_scripted(Tracker, case, True)
    assert check_rle_results(plain.results, rle.results) > 0
    for a, b in zip(plain.tracks, rle.tracks):                      # Track.mask is untouched
        assert a.id == b.id and torch.equal(a.mask, b.mask)
    fa = write_results(plain.results, str(tmp_path / "a"), "seq")
    fb = write_results(rle.results, str(tmp_path / "b"), "seq")
    assert open(fa, "rb").read() == open(fb, "rb").read()


def test_mask_rle_entry_point_rejects_bad_arguments():
    """-1 NULL pointer, -2 bad shape or short workspace, 0 for T == 0 (checks run before anything touches the
    device); the size queries"""
    from trackformer_b200 import ext
    ext.load()
    lib = ctypes.CDLL(ext.library_path())
    ws = lib.tfb200_mask_rle_workspace_bytes
    ws.restype, ws.argtypes = ctypes.c_size_t, [ctypes.c_int] * 3
    mx = lib.tfb200_mask_rle_max_bytes
    mx.restype, mx.argtypes = ctypes.c_int64, [ctypes.c_int] * 3
    f = lib.tfb200_mask_rle_i32
    f.restype = ctypes.c_int
    f.argtypes = ([ctypes.c_void_p] * 2 + [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                                                  ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p])
    assert ws(0, 8, 1) == 0 and ws(8, 8, -1) == 0 and ws(1 << 15, 1 << 14, 1) == 0
    assert ws(8, 8, 1) >= 4 * 64 * 3 and ws(800, 1333, 100) > ws(800, 1333, 1)
    assert mx(3, 4, 1) == 1 * (24 + 1) and mx(1080, 1920, 100) == 5 * (2 * 1080 * 1920 + 100)
    buf = (ctypes.c_int32 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    big = ws(8, 8, 2)
    assert f(None, p, 8, 8, 2, p, big, p, p, 100, None) == -1
    assert f(p, None, 8, 8, 2, p, big, p, p, 100, None) == -1
    assert f(p, p, 8, 8, 2, None, big, p, p, 100, None) == -1
    assert f(p, p, 8, 8, 2, p, big, None, p, 100, None) == -1
    assert f(p, p, 8, 8, 2, p, big, p, None, 100, None) == -1
    assert f(p, p, 0, 8, 2, p, big, p, p, 100, None) == -2                    # H
    assert f(p, p, 8, -1, 2, p, big, p, p, 100, None) == -2                   # W
    assert f(p, p, 8, 8, -1, p, big, p, p, 100, None) == -2                   # T
    assert f(p, p, 1 << 15, 1 << 14, 2, p, big, p, p, 100, None) == -2        # H * W > 2^28
    assert f(p, p, 8, 8, 2, p, big, p, p, -1, None) == -2                     # capacity
    assert f(p, p, 8, 8, 2, p, big - 1, p, p, 100, None) == -2                # workspace too small
    assert f(p, p, 8, 8, 0, p, 0, p, p, 0, None) == 0
