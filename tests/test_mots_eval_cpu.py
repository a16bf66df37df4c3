"""MOTS evaluation on the CPU suite.

The oracle (tests/mots_eval_reference.py) is pinned on the worked example and hand vectors at each boundary of the
definition; then csrc/mots_eval_core.h -- the routines csrc/mots_eval.cu's kernels are compiled from, built here by g++
with one "thread" (tests/host_build/mots_eval_host.cpp) -- is compared with the oracle through the product's packing
(`get_mots_accum`) and summary (`summarize`).  Also: the string decoder against `mots.decode_counts`, the MOTS20 file
round trip, the pickle round trip, and every error class.  The CUDA build is compared in tests/test_mots_eval_gpu.py."""
import ctypes
import pickle

import numpy as np
import pytest
import torch

import host_twin
import mots_eval_fixtures as msf
import mots_eval_reference as ref
from trackformer_b200 import mots, mots_eval

INTS = ("num_unique_objects", "mostly_tracked", "partially_tracked", "mostly_lost", "num_detections",
        "num_false_positives", "num_misses", "num_switches", "num_fragmentations", "num_ignored")


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    lib = host_twin.build("mots_eval_host", tmp_path_factory.mktemp("mots_eval"))
    i32, i64, vp = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p
    lib.tfb200_mots_eval_host_workspace_bytes.argtypes = [i32, i32, i32, i64, i64, i64, i32, i32, i64, i64, i64]
    lib.tfb200_mots_eval_host_workspace_bytes.restype = ctypes.c_size_t
    lib.tfb200_mots_eval_host.argtypes = [vp] * 9 + [i32, i32, i32, i64, i64, i64, i32, i32, i64, i64, i64, vp,
                                                     ctypes.c_size_t, vp]
    lib.tfb200_mots_eval_host.restype = ctypes.c_int
    lib.tfb200_mots_decode_host.argtypes = [vp, i64, i32, i32, vp, i64]
    lib.tfb200_mots_decode_host.restype = i64
    return lib


def host_counters(lib, accums, names=None):
    """The device algorithm run on the host through the product's packing: out [S, 16 + 11], checked as the product
    checks the device's."""
    buf, offsets, z = mots_eval._pack(accums)
    args = mots_eval._entry_args(z)
    ws = np.zeros(lib.tfb200_mots_eval_host_workspace_bytes(*args) + 256, np.uint8)
    out = np.zeros(z["S"] * (16 + mots_eval._XSLOTS), np.int64)
    ws_ptr = (ws.ctypes.data + 255) // 256 * 256
    rc = lib.tfb200_mots_eval_host(*[buf.ctypes.data + o for o in offsets], *args, ws_ptr, ws.nbytes - 256,
                                   out.ctypes.data)
    assert rc == 0
    return mots_eval.check_counters(out, z, names)


def oracle_counts(results, gt, n_frames):
    return ref.counts(*ref.accumulate(results, gt, n_frames))


def check_summary(summary, expected):
    """expected: {name: oracle metrics}; integer columns exactly, ratios within 1e-12."""
    assert list(summary.index) == list(expected)
    for name, want in expected.items():
        for col in mots_eval.COLUMNS:
            got = summary[col][name]
            if col in INTS:
                assert int(got) == int(want[col]), (name, col, got, want[col])
            elif np.isnan(want[col]):
                assert np.isnan(got), (name, col, got)
            else:
                assert abs(float(got) - float(want[col])) <= 1e-12, (name, col, got, want[col])


def run_host(lib, named):
    """named {name: (results, gt, n_frames)}: host build vs oracle; returns (summary, out, expected counts)"""
    accums = [mots_eval.get_mots_accum(r, g, n) for r, g, n in named.values()]
    out = host_counters(lib, accums, list(named))
    summary, _ = mots_eval.summarize(accums, list(named), out)
    counts = {n: oracle_counts(*v) for n, v in named.items()}
    check_summary(summary, ref.evaluate(counts))
    for s, c in enumerate(counts.values()):                 # sum of d bit for bit
        assert out[s, 15:16].view(np.float64)[0] == c["sum_d"]
    return summary, out, counts


# ---- hand vectors (H x W dense masks, given as RLEs) ----

def _m(h, w, cols=(), rows=None, pixels=()):
    a = np.zeros((h, w), bool)
    for c in cols:
        a[slice(None) if rows is None else list(rows), c] = True
    for r, c in pixels:
        a[r, c] = True
    return a


def _seq(h, w, frames_gt, frames_ign, frames_hyp):
    """frames_gt[f] {oid: mask}, frames_ign[f] [mask], frames_hyp[f] {tid: mask} -> (results, gt, n_frames)"""
    gt, results = {}, {}
    for f, objs in enumerate(frames_gt):
        for o, m in objs.items():
            gt.setdefault(o, {})[f] = {"mask": mots.encode(m), "class_id": 2}
        for k, m in enumerate(frames_ign[f]):
            gt.setdefault(10000 + k, {})[f] = {"mask": mots.encode(m), "class_id": 10}
        for t, m in frames_hyp[f].items():
            results.setdefault(t, {})[f] = {"mask": mots.encode(m)}
    return results, gt, len(frames_gt)


def worked_example():
    H, W = 4, 6
    A, B = _m(H, W, (0, 1)), _m(H, W, (3, 4))
    return _seq(H, W, [{1: A, 2: B}, {1: A, 2: B}], [[_m(H, W, (5,))], []],
                [{"t0": _m(H, W, (0, 1), range(3)), "t1": _m(H, W, (2, 3)), "t2": _m(H, W, (5,), range(3))},
                 {"t1": _m(H, W, (0, 1)), "t0": _m(H, W, (3, 4), range(2))}])


def test_oracle_worked_example():
    c = oracle_counts(*worked_example())
    m = ref.metrics(c)
    tp = c["matches"] + c["switches"]
    assert (tp, c["fp"], c["misses"], c["switches"], c["sum_d"], c["removed"]) == (3, 1, 1, 1, 0.75, 1)
    assert (m["motsa"], m["smotsa"], m["motsp"], m["recall"], m["precision"]) == (0.25, 0.0625, 0.75, 0.75, 0.75)
    assert (m["idf1"], m["idp"], m["idr"]) == (0.5, 0.5, 0.5)
    assert (c["gt"], c["mt"], c["pt"], c["ml"], c["fm"]) == (2, 1, 1, 0, 0)


def boundary_scenes():
    """one frame each, 4 x 6: IoU exactly 0.5 (candidate) and 2 inter = union - 1 (not); 2 |h & ign| = |h| (kept)
    and = |h| + 1 (removed); an empty hypothesis; frames without GT or without hypotheses; a candidate mostly inside
    an ignore region."""
    H, W = 4, 6
    g = _m(H, W, (0,))                                            # 4 pixels
    half = _m(H, W, (0,), range(2))                               # inter 2, union 4
    under = _m(H, W, (0,), range(2), pixels=[(0, 1)])             # inter 2, union 5
    ign = _m(H, W, (4, 5))
    keep_h = _m(H, W, (3, 4), range(2))                           # 4 pixels, 2 in the ignore region
    drop_h = _m(H, W, (3, 4), range(2), pixels=[(2, 4)])          # 5 pixels, 3 in it
    cand_in_ign = _m(H, W, (4, 5), range(3))                      # IoU 6 / 8 with a GT there, all in the ignore
    return {
        "iou_half": _seq(H, W, [{1: g}], [[]], [{7: half}]),
        "iou_under": _seq(H, W, [{1: g}], [[]], [{7: under}]),
        "ign_equal": _seq(H, W, [{1: g}], [[ign]], [{7: keep_h}]),
        "ign_over": _seq(H, W, [{1: g}], [[ign]], [{7: drop_h}]),
        "empty_hyp": _seq(H, W, [{1: g}], [[ign]], [{7: np.zeros((H, W), bool)}]),
        "no_gt": _seq(H, W, [{}, {1: g}], [[], []], [{7: g}, {}]),
        "cand_in_ign": _seq(H, W, [{1: _m(H, W, (4, 5))}], [[_m(H, W, (3,))]], [{7: cand_in_ign}]),
    }


def test_oracle_boundaries():
    got = {n: oracle_counts(*v) for n, v in boundary_scenes().items()}
    assert (got["iou_half"]["matches"], got["iou_half"]["sum_d"]) == (1, 0.5)
    assert (got["iou_under"]["matches"], got["iou_under"]["fp"]) == (0, 1)
    assert (got["ign_equal"]["fp"], got["ign_equal"]["removed"]) == (1, 0)
    assert (got["ign_over"]["fp"], got["ign_over"]["removed"], got["ign_over"]["num_predictions"]) == (0, 1, 0)
    assert (got["empty_hyp"]["fp"], got["empty_hyp"]["removed"]) == (1, 0)
    assert (got["no_gt"]["fp"], got["no_gt"]["misses"]) == (1, 1)
    assert (got["cand_in_ign"]["matches"], got["cand_in_ign"]["removed"]) == (1, 0)


# ---- the host build of the kernels' source against the oracle ----

def test_host_build_worked_example_and_boundaries(host_lib):
    summary, out, _ = run_host(host_lib, {"example": worked_example(), **boundary_scenes()})
    assert summary["smotsa"]["example"] == 0.0625 and summary["num_ignored"]["example"] == 1
    assert out[0, 16 + mots_eval._XINTERVALS] > 0


def _random_counts(rng, n):
    """run lengths covering n pixels: long runs, one-run masks, many short runs (negative deltas)"""
    kind = rng.integers(0, 4)
    if kind == 0:
        return np.asarray([n])
    if kind == 1:
        return np.asarray([0, n])
    k = int(rng.integers(2, 400 if kind == 2 else 8))
    cuts = np.sort(rng.choice(np.arange(1, n), size=min(k, n - 1), replace=False))
    c = np.diff(np.concatenate(([0], cuts, [n])))
    if rng.random() < 0.5:
        c = np.concatenate(([0], c))
    return c


def test_decoder_equals_decode_counts(host_lib):
    rng = np.random.default_rng(5)
    for _ in range(300):
        h, w = int(rng.integers(1, 200)), int(rng.integers(1, 300))
        cnts = _random_counts(rng, h * w).astype(np.int64)
        s = mots._string(cnts)
        np.testing.assert_array_equal(mots.decode_counts(s), cnts)
        want = np.cumsum(np.concatenate(([0], cnts)))
        iv = np.stack([want[1:-1:2], want[2::2]], 1) if len(cnts) > 1 else np.zeros((0, 2), np.int64)
        iv = iv[iv[:, 1] > iv[:, 0]]
        buf = np.frombuffer(s, np.uint8).copy()
        out = np.zeros(2 * max(1, len(iv)), np.int32)
        n = host_lib.tfb200_mots_decode_host(buf.ctypes.data, len(buf), h, w, out.ctypes.data, len(iv))
        assert n == len(iv)
        np.testing.assert_array_equal(out[:2 * n].reshape(-1, 2), iv)


def test_decoder_rejects_bad_strings(host_lib):
    def dec(s, h=4, w=6):
        buf = np.frombuffer(s, np.uint8).copy() if s else np.zeros(1, np.uint8)
        out = np.zeros(64, np.int32)
        return host_lib.tfb200_mots_decode_host(buf.ctypes.data, len(s), h, w, out.ctypes.data, 32)
    good = mots.encode(_m(4, 6, (1, 3)))["counts"]
    assert dec(good) == 2
    assert dec(good[:-1]) == -1                                # runs short of H x W
    assert dec(good + b"0") == -1                              # a zero delta repeats the count two back: past H x W
    assert dec(good + b"1") == -1                              # runs past H x W
    assert dec(b"") == -1
    assert dec(good[:-1] + b"h") == -1                         # a last value cut short (continuation bit)
    assert dec(b"~" + good[1:]) == -1                          # a character outside '0' .. 'o'
    assert dec(b"hhhhhhh0") == -1                              # a value of more than 7 characters
    assert dec(mots._string(np.asarray([4, 8, 2, -2, 12]))) == -1   # a negative count


@pytest.mark.parametrize("seed", range(12))
def test_host_build_matches_oracle_on_synthetic_sequences(host_lib, seed):
    rng = np.random.default_rng(seed)
    style = "fragmented" if seed % 3 == 2 else "person"
    named = {}
    for k in range(3):                                         # several sequences, different sizes, in one call
        size = [(96, 160), (64, 128), (120, 200)][(seed + k) % 3]
        r, g = msf.scene(100 * seed + k, n_frames=int(rng.integers(5, 25)), n_objects=int(rng.integers(1, 8)),
                         size=size, style=style, p_switch=float(rng.uniform(0, 0.1)))
        named[f"seq{k}"] = (r, g, max([f + 1 for tr in g.values() for f in tr], default=1))
    run_host(host_lib, named)


def test_host_build_frames_past_the_end_and_other_classes(host_lib):
    r, g = msf.scene(3, n_frames=12)
    r[999] = {11: {"mask": msf.rle([], 96, 160)}, 40: {"mask": msf.rle([[0, 5]], 96, 160)}}
    g[55] = {2: {"mask": msf.rle([[0, 5]], 96, 160), "class_id": 1}}    # a car: dropped
    named = {"short": (r, g, 10)}
    run_host(host_lib, named)


# ---- files, pickling, errors ----

def test_load_results_round_trips_byte_for_byte(tmp_path):
    r, g = msf.scene(4, n_frames=8)
    path = mots.write_results(r, str(tmp_path / "a"), "MOTS20-02")
    back = mots.load_results(path)
    assert list(back) == list(r)
    again = mots.write_results(back, str(tmp_path / "b"), "MOTS20-02")
    assert open(path, "rb").read() == open(again, "rb").read()
    for t, tr in r.items():
        for f, d in tr.items():
            assert back[t][f]["mask"]["counts"] == d["mask"]["counts"] and back[t][f]["class_id"] == 2


def test_gt_file_and_dict_give_one_accumulator(tmp_path):
    r, g = msf.scene(6, n_frames=10)
    path = tmp_path / "gt.txt"
    with open(path, "w") as f:                                 # GT file order: frame, then the dict's id order
        for fr in range(10):
            for i, tr in g.items():
                if fr in tr:
                    m = tr[fr]["mask"]
                    f.write(f"{fr + 1} {i + 1} {tr[fr]['class_id']} {m['size'][0]} {m['size'][1]} "
                            f"{m['counts'].decode()}\n")
    a = mots_eval.get_mots_accum(r, g, 10)
    b = mots_eval.get_mots_accum(r, str(path), 10)
    c = pickle.loads(pickle.dumps(a))
    for x in (b, c):
        for k in ("frame_mask", "mask_id", "mask_size", "str_off", "chars", "gt_ids", "track_ids"):
            np.testing.assert_array_equal(getattr(a, k), getattr(x, k))


def test_bool_masks_pack_like_rles():
    r, g = msf.scene(7, n_frames=6)
    rb, _ = msf.scene(7, n_frames=6, as_rle=False)
    a, b = mots_eval.get_mots_accum(r, g, 6), mots_eval.get_mots_accum(rb, g, 6)
    np.testing.assert_array_equal(a.chars, b.chars)
    np.testing.assert_array_equal(a.str_off, b.str_off)


def _error_case(kind):
    H, W = 4, 6
    A, B = _m(H, W, (0, 1)), _m(H, W, (3, 4))
    fr_gt = [{1: A}, {1: A, 2: B}, {1: A, 2: B}]
    fr_ign, fr_hyp = [[], [], []], [{5: A}, {5: A, 6: B}, {5: A, 6: B}]
    if kind == "gt_overlap":
        fr_ign[1] = [_m(H, W, (4, 5))]
    if kind == "hyp_overlap":
        fr_hyp[2] = {5: A, 6: _m(H, W, (1, 2))}
    results, gt, n = _seq(H, W, fr_gt, fr_ign, fr_hyp)
    if kind == "size":
        results[6][1]["mask"] = mots.encode(np.zeros((4, 7), bool))
    if kind == "malformed":
        gt[2][2]["mask"] = {"size": [H, W], "counts": b"0\x7f"}
    if kind == "short":
        gt[2][1]["mask"] = {"size": [H, W], "counts": mots.encode(B)["counts"][:-1]}
    return results, gt, n


@pytest.mark.parametrize("kind, frame, what", [
    ("gt_overlap", 1, "GT masks"), ("hyp_overlap", 2, "result masks overlap"), ("size", 1, "size differs"),
    ("malformed", 2, "malformed"), ("short", 1, "malformed")])
def test_every_error_class_raises_with_sequence_and_frame(host_lib, kind, frame, what):
    ok = _seq(4, 6, [{1: _m(4, 6, (0,))}], [[]], [{}])
    accums = [mots_eval.get_mots_accum(*ok), mots_eval.get_mots_accum(*_error_case(kind))]
    with pytest.raises(ValueError, match=rf"sequence MOTS20-11: frame {frame}: .*{what}"):
        host_counters(host_lib, accums, ["MOTS20-02", "MOTS20-11"])


def test_duplicate_frame_and_id_in_a_file_raises(tmp_path):
    p = tmp_path / "MOTS20-05.txt"
    p.write_text("1 1 2 4 6 8<0\n2 1 2 4 6 8<0\n2 1 2 4 6 8<0\n")
    with pytest.raises(ValueError, match="MOTS20-05.txt: frame 2: duplicate id 1"):
        mots.load_results(str(p))
    with pytest.raises(ValueError, match="duplicate"):
        mots_eval.get_mots_accum({}, str(p), 3)


def test_evaluation_needs_cuda(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    acc = mots_eval.get_mots_accum(*worked_example())
    with pytest.raises(RuntimeError, match="CUDA"):
        mots_eval.evaluate_mots_accums([acc], ["s"])


def test_str_summary_columns(host_lib):
    named = {"MOTS20-02": (*msf.scene(8, n_frames=10), 10), "MOTS20-05": (*msf.scene(9, n_frames=12), 12)}
    accums = [mots_eval.get_mots_accum(*v) for v in named.values()]
    summary, text = mots_eval.summarize(accums, list(named), host_counters(host_lib, accums))
    lines = text.splitlines()
    assert lines[0].split() == ["sMOTSA", "MOTSA", "MOTSP", "IDF1", "IDP", "IDR", "Rcll", "Prcn", "GT", "MT", "PT",
                                "ML", "TP", "FP", "FN", "IDs", "FM", "Ign"]
    assert [ln.split()[0] for ln in lines[1:]] == ["MOTS20-02", "MOTS20-05", "OVERALL"]
    assert lines[3].split()[1] == f"{summary['smotsa']['OVERALL']:.1%}"
