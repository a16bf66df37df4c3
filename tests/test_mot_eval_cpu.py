"""MOT evaluation on the CPU suite.

The oracle (tests/mot_eval_reference.py) is pinned on hand-worked vectors; then csrc/mot_eval_core.h -- the routines
csrc/mot_eval.cu's kernels are compiled from, built here by g++ with one "thread" (tests/host_build/mot_eval_host.cpp)
-- is compared with the oracle on seeded synthetic sequences through the product's own packing (`get_mot_accum`) and
summary (`summarize`).  Also: both GT box formats, the pickle round trip, the C entry's argument checks and the
rendering of `str_summary`.  The CUDA build of the same source is compared in tests/test_mot_eval_gpu.py."""
import ctypes
import pickle

import numpy as np
import pytest
import torch

import host_twin
import mot_eval_fixtures as mf
import mot_eval_reference as ref
from trackformer_b200 import mot_eval

INTS = ("num_unique_objects", "mostly_tracked", "partially_tracked", "mostly_lost", "num_false_positives",
        "num_misses", "num_switches", "num_fragmentations")


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    lib = host_twin.build("mot_eval_host", tmp_path_factory.mktemp("mot_eval"))
    i32, i64, vp = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p
    lib.tfb200_mot_eval_host_workspace_bytes.argtypes = [i32, i32, i64, i64, i64, i32, i32, i64]
    lib.tfb200_mot_eval_host_workspace_bytes.restype = ctypes.c_size_t
    lib.tfb200_mot_eval_host.argtypes = [vp] * 7 + [i32, i32, i64, i64, i64, i32, i32, i64, vp, ctypes.c_size_t, vp]
    lib.tfb200_mot_eval_host.restype = ctypes.c_int
    return lib


def host_counters(lib, accums, pair_cap=None):
    """The device algorithm run on the host, through the product's packing: out [S, 16]."""
    buf, offsets, z = mot_eval._pack(accums)
    cap = z["products"] if pair_cap is None else pair_cap
    ws = np.zeros(lib.tfb200_mot_eval_host_workspace_bytes(z["S"], z["F"], z["n_gt"], z["n_trk"], z["tp_cells"],
                                                           z["max_obj"], z["max_hyp"], cap) + 256, np.uint8)
    out = np.zeros((z["S"], 16), np.int64)
    base = buf.ctypes.data
    ws_ptr = (ws.ctypes.data + 255) // 256 * 256
    rc = lib.tfb200_mot_eval_host(*[base + o for o in offsets], z["S"], z["F"], z["n_gt"], z["n_trk"],
                                  z["tp_cells"], z["max_obj"], z["max_hyp"], cap, ws_ptr, ws.nbytes - 256,
                                  out.ctypes.data)
    assert rc == 0
    return out


def oracle_counts(results, frames):
    return ref.counts(ref.accumulate(results, [fr["gt"] for fr in frames]))


def check_summary(summary, expected):
    """expected: {name: oracle metrics}; integer columns exactly, ratios within 1e-12."""
    assert list(summary.index) == list(expected)
    for name, want in expected.items():
        for col in mot_eval.COLUMNS:
            got = summary[col][name]
            if col in INTS:
                assert int(got) == int(want[col]), (name, col, got, want[col])
            elif np.isnan(want[col]):
                assert np.isnan(got), (name, col, got)
            else:
                assert abs(float(got) - float(want[col])) <= 1e-12, (name, col, got, want[col])


# ---- the oracle on hand-worked vectors ----

def test_oracle_three_frame_vector():
    nan = np.nan
    acc = ref.Accumulator()
    acc.update([1, 2], [1, 2, 3], [[0.1, nan, 0.3], [0.5, 0.2, 0.3]])
    acc.update([1, 2], [1], [[0.2], [0.4]])
    acc.update([1, 2], [1, 3], [[0.6, 0.2], [0.1, 0.6]])
    ev = [(f, k, o, h, None if np.isnan(d) else round(d, 12)) for f, k, o, h, d in acc.events]
    assert ev == [(0, "MATCH", 1, 1, 0.1), (0, "MATCH", 2, 2, 0.2), (0, "FP", None, 3, None),
                  (1, "MATCH", 1, 1, 0.2), (1, "MISS", 2, None, None),
                  (2, "MATCH", 1, 1, 0.6), (2, "SWITCH", 2, 3, 0.6)]
    m = ref.metrics(ref.counts(acc))
    assert m["mota"] == 0.5 and abs(m["motp"] - 0.34) < 1e-15
    assert (m["num_false_positives"], m["num_misses"], m["num_switches"]) == (1, 1, 1)
    assert ref.counts(acc)["idtp"] == 5 and abs(m["idf1"] - 5 / 6) < 1e-15


def test_oracle_prefers_more_pairs_over_smaller_sum():
    nan = np.nan
    acc = ref.Accumulator()
    acc.update(["a", "b"], ["x", "y"], [[0.1, 0.3], [0.3, nan]])     # (a, x) alone has the least sum
    assert sorted((k, o, h) for _, k, o, h, _ in acc.events) == [("MATCH", "a", "y"), ("MATCH", "b", "x")]


def test_iou_exactly_half_is_valid():
    d = ref.iou_distance(ref.to_xywh([[0, 0, 2, 1]]), ref.to_xywh([[0, 0, 1, 1]]))
    assert d[0, 0] == 0.5


# ---- the host build of the kernels' source against the oracle ----

def _run_both(host_lib, named):
    accums = [mot_eval.get_mot_accum(r, fr) for r, fr in named.values()]
    out = host_counters(host_lib, accums)
    summary, _ = mot_eval.summarize(accums, list(named), out)
    expected = ref.evaluate({n: oracle_counts(r, fr) for n, (r, fr) in named.items()})
    check_summary(summary, expected)
    return summary, out


def _frames(*gts):
    return [{"gt": {k: np.asarray(v, np.float32) for k, v in g.items()}} for g in gts]


def _bb(*b):
    return {"bbox": np.asarray(b, np.float32)}


def hand_scenes():
    """"larger": one frame, no previous partners.  Objects a = 1, b = 2; hypotheses x = 8, y = 7 with d(a, x) ~ 0.001,
    d(a, y) ~ 0.46, d(b, x) ~ 0.46, (b, y) invalid: (a, x) alone has the least sum, but the two-pair matching
    (a, y), (b, x) must win.  "half": IoU exactly 0.5 is a match."""
    return {"larger": ({7: {0: _bb(-3, 0, 7, 10)}, 8: {0: _bb(0.01, 0, 10, 10)}},
                       _frames({1: [0, 0, 10, 10], 2: [3, 0, 13, 10]})),
            "half": ({7: {0: _bb(0, 0, 1, 1)}}, _frames({1: [0, 0, 2, 1]}))}


def check_hand_scenes(summary):
    s = summary.loc["larger"]
    assert (s["num_misses"], s["num_false_positives"], s["num_switches"], s["recall"]) == (0, 0, 0, 1.0)
    assert 0.45 < s["motp"] < 0.47                            # the two-pair matching, not (a, x) at d ~ 0.001
    s = summary.loc["half"]
    assert (s["num_misses"], s["num_false_positives"], s["motp"]) == (0, 0, 0.5)


def test_host_build_iou_half_and_larger_matching(host_lib):
    summary, _ = _run_both(host_lib, hand_scenes())
    check_hand_scenes(summary)


def test_host_build_float32_width_moves_a_pair_across_the_threshold(host_lib):
    """GT [x1, 0, X, 1] with X - x1 rounding to X in float32, so x1 + fl32(X - x1) != X, against a hypothesis
    [0, 0, X, yb]: with yb just below 2 the exact extents give IoU >= 0.5 and the float32 width gives less."""
    def dist(g, h, f32):
        conv = ref.to_xywh if f32 else (lambda b: np.r_[b[:2], b[2:] - b[:2]][None])
        if not f32:
            g, h = g.astype(np.float64), h.astype(np.float64)
        return ref.iou_distance(conv(g), conv(h))[0, 0]

    x1, found = np.float32(0.45), None
    for k in range(1, 2000):
        X = np.float32(2 ** 23 + k)                  # spacing 1: X - x1 rounds to X
        yb0 = np.float32(2 * (np.float64(X) - np.float64(x1)) / np.float64(X))
        for yb in (yb0, np.nextafter(yb0, np.float32(0)), np.nextafter(yb0, np.float32(3))):
            g, h = np.asarray([x1, 0, X, 1], np.float32), np.asarray([0, 0, X, yb], np.float32)
            if np.isnan(dist(g, h, True)) != np.isnan(dist(g, h, False)):
                found = g, h
                break
        if found:
            break
    assert found, "no pair crosses the threshold"
    g, h = found
    assert np.float64(g[0]) + np.float64(g[2] - g[0]) != np.float64(g[2])
    summary, _ = _run_both(host_lib, {"s": ({3: {0: {"bbox": h}}}, _frames({1: g}))})
    assert summary["num_misses"]["s"] == (1 if np.isnan(dist(g, h, True)) else 0)


def test_host_build_empty_frames_and_a_sequence_without_tracks(host_lib):
    gt1 = {1: [0, 0, 10, 10], 2: [20, 0, 30, 10]}
    frames = _frames({}, gt1, gt1, {}, gt1, {1: [1, 0, 11, 10]})
    results = {5: {1: _bb(0, 0, 10, 10), 2: _bb(0, 0, 10, 10), 3: _bb(50, 50, 60, 60), 5: _bb(1, 0, 11, 10),
                   99: _bb(0, 0, 1, 1)},
               6: {2: _bb(20, 0, 30, 10)}}
    named = {"a": (results, frames), "b": ({}, _frames(gt1, {}, gt1)), "c": ({}, _frames({}, {}))}
    summary, _ = _run_both(host_lib, named)
    assert summary["num_misses"]["b"] == 4 and summary["num_false_positives"]["a"] == 1


def test_host_build_fragmentation_after_a_gap(host_lib):
    g = {1: [0, 0, 10, 10]}
    frames = _frames(g, g, {}, g, g, g, g)
    results = {4: {0: _bb(0, 0, 10, 10), 4: _bb(0, 0, 10, 10), 6: _bb(0, 0, 10, 10)}}   # hit, miss, -, miss, hit ...
    summary, _ = _run_both(host_lib, {"s": (results, frames)})
    assert summary["num_fragmentations"]["s"] == 2


SEEDS = list(range(30))


@pytest.mark.parametrize("seed", SEEDS)
def test_host_build_matches_oracle_on_synthetic_scenes(host_lib, seed):
    rng = np.random.default_rng(1000 + seed)
    kw = dict(n_frames=int(rng.integers(20, 60)), n_objects=int(rng.integers(3, 25)),
              p_swap=float(rng.uniform(0, 0.05)), p_dup=float(rng.uniform(0, 0.2)), fp_rate=float(rng.uniform(0, 2)))
    if seed % 3 == 2:                                        # crowded: residual components of several boxes
        kw.update(width=120.0, height=160.0, n_objects=int(rng.integers(8, 30)))
    _run_both(host_lib, {f"seq{seed}": mf.scene(seed, **kw), "other": mf.scene(seed + 100, n_frames=15)})


def test_host_build_crowded_frames_match_oracle(host_lib):
    summary, out = _run_both(host_lib, {"clumps": mf.clumps(1, n_frames=6)})
    assert out[0, 11] >= 3 and out[0, 12] >= 3


def test_host_build_reports_a_small_pair_buffer(host_lib):
    accums = [mot_eval.get_mot_accum(*mf.scene(s, n_frames=10)) for s in (1, 2)]
    full = host_counters(host_lib, accums)
    small = host_counters(host_lib, accums, pair_cap=int(full[:, 1].sum()) - 1)
    assert (small[:, 0] == 1).all() and (small[:, 1] == full[:, 1]).all()
    exact = host_counters(host_lib, accums, pair_cap=int(full[:, 1].sum()))
    assert (exact == full).all()


# ---- packing, pickling, entry checks, rendering ----

def test_get_mot_accum_gt_formats_and_pickle():
    results, frames = mf.scene(3, n_frames=12)
    collated = mf.scene(3, n_frames=12, gt_box=lambda b: torch.from_numpy(np.asarray(b))[None])[1]
    assert isinstance(next(iter(collated[1]["gt"].values())), torch.Tensor)
    a, b = mot_eval.get_mot_accum(results, frames), mot_eval.get_mot_accum(results, collated)
    c = pickle.loads(pickle.dumps(a))
    for x in (b, c):
        for k in ("frame_obj", "obj_id", "obj_box", "frame_hyp", "hyp_id", "hyp_box", "gt_ids", "track_ids"):
            np.testing.assert_array_equal(getattr(a, k), getattr(x, k))
    # rows follow the gt dict order and the order results lists its tracks; x, y, w, h in float32
    f = 5
    gt = frames[f]["gt"]
    rows = slice(a.frame_obj[f], a.frame_obj[f + 1])
    np.testing.assert_array_equal(a.gt_ids[a.obj_id[rows]], list(gt))
    np.testing.assert_array_equal(a.obj_box[rows], ref.to_xywh(list(gt.values())))
    tids = [t for t, tr in results.items() if f in tr]
    hrows = slice(a.frame_hyp[f], a.frame_hyp[f + 1])
    np.testing.assert_array_equal(a.track_ids[a.hyp_id[hrows]], tids)
    np.testing.assert_array_equal(a.hyp_box[hrows], ref.to_xywh([results[t][f]["bbox"] for t in tids]))
    # frames past the loader's end are ignored
    short = mot_eval.get_mot_accum(results, frames[:4])
    assert short.num_frames == 4 and short.frame_hyp[-1] == sum(f < 4 for tr in results.values() for f in tr)


def test_str_summary_columns_and_formats(host_lib):
    named = {"MOT17-02": mf.scene(7, n_frames=20), "MOT17-04": mf.scene(8, n_frames=25)}
    accums = [mot_eval.get_mot_accum(r, fr) for r, fr in named.values()]
    summary, text = mot_eval.summarize(accums, list(named), host_counters(host_lib, accums))
    lines = text.splitlines()
    assert lines[0].split() == ["IDF1", "IDP", "IDR", "Rcll", "Prcn", "GT", "MT", "PT", "ML", "FP", "FN", "IDs",
                                "FM", "MOTA", "MOTP"]
    assert [ln.split()[0] for ln in lines[1:]] == ["MOT17-02", "MOT17-04", "OVERALL"]
    row = lines[3].split()[1:]
    s = summary.loc["OVERALL"]
    assert row[0] == f"{s['idf1']:.1%}" and row[13] == f"{s['mota']:.1%}" and row[14] == f"{s['motp']:.3f}"
    assert row[5] == str(int(s["num_unique_objects"])) and row[9] == str(int(s["num_false_positives"]))
    assert summary["mota"]["OVERALL"] == s["mota"]                   # engine.py's access pattern
    no_overall, _ = mot_eval.summarize(accums, list(named), host_counters(host_lib, accums), generate_overall=False)
    assert list(no_overall.index) == list(named)


def test_entry_rejects_bad_arguments():
    from trackformer_b200 import ext
    lib = ctypes.CDLL(ext.library_path())
    i32, i64, vp = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p
    ws = lib.tfb200_mot_eval_workspace_bytes
    ws.argtypes, ws.restype = [i32, i32, i64, i64, i64, i32, i32, i64], ctypes.c_size_t
    f = lib.tfb200_mot_eval_f32
    f.argtypes = [vp] * 7 + [i32, i32, i64, i64, i64, i32, i32, i64, vp, ctypes.c_size_t, vp, vp]
    f.restype = ctypes.c_int
    good = (1, 4, 3, 5, 15, 2, 3, 10)
    n = ws(*good)
    assert n > 0
    for bad in ((0, 4, 3, 5, 15, 2, 3, 10), (1, -1, 3, 5, 15, 2, 3, 10), (1, 4, -3, 5, 15, 2, 3, 10),
                (1, 4, 3, 5, 15, -2, 3, 10), (1, 4, 3, 5, 15, 2, 3, -1), (1, 4, 2 ** 31, 5, 15, 2, 3, 10),
                (1, 4, 3, 5, 15, 65536, 65536, 10)):
        assert ws(*bad) == 0
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, vp).value
    assert f(None, *[p] * 6, *good, p, n, p, None) == -1
    assert f(*[p] * 7, *good, None, n, p, None) == -1
    assert f(*[p] * 7, *good, p, n, None, None) == -1
    assert f(*[p] * 7, 0, 4, 3, 5, 15, 2, 3, 10, p, n, p, None) == -2
    assert f(*[p] * 7, *good, p, n - 1, p, None) == -2


def test_evaluation_needs_cuda(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    acc = mot_eval.get_mot_accum(*mf.scene(1, n_frames=3))
    with pytest.raises(RuntimeError, match="CUDA"):
        mot_eval.evaluate_mot_accums([acc], ["s"])
