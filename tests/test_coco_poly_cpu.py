"""Polygon ground-truth masks on the CPU suite.

The oracle (tests/coco_poly_reference.py, pycocotools' rleFrPoly / frBbox / frPyObjects / merge restated in Python) is
pinned on hand values; then csrc/coco_poly_core.h -- the routines csrc/coco_poly.cu's kernels are compiled from,
built here by g++ -ffp-contract=off with one "thread" (tests/host_build/coco_poly_host.cpp) -- is compared with it run
for run through the product's packing (`coco_masks.pack_polygons`) and error reporting (`coco_masks.check_sizes`).
The CUDA build is compared in tests/test_coco_poly_gpu.py."""
import ctypes
from fractions import Fraction

import numpy as np
import pytest

import coco_poly_fixtures as pf
import coco_poly_reference as ref
import eval_consistency_fixtures as ef
import host_twin
from trackformer_b200 import coco_eval, coco_masks, mots



@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    lib = host_twin.build("coco_poly_host", tmp_path_factory.mktemp("coco_poly"))
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    geo = [vp] * 5 + [i32, i32, i64]
    lib.tfb200_coco_poly_count_host.argtypes = geo + [vp, vp, vp]
    lib.tfb200_coco_poly_runs_host.argtypes = geo + [vp, i64, vp, vp]
    lib.tfb200_coco_rle_runs_host.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp]
    lib.tfb200_coco_masks_u8_host.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp, vp]
    return lib


def _p(a):
    return a.ctypes.data


def host_runs(lib, segs, hw, names=None):
    """The device algorithm on the host through the product's packing: (run_off, runs int64 [R, 2])."""
    names = names or [f"annotation {i}" for i in range(len(segs))]
    z = coco_masks.pack_polygons(segs, hw, names)
    P, A, E = coco_masks.geometry(z)
    geo = [_p(z[k]) for k in ("xy", "part_off", "part_ann", "ann_part", "ann_hw")] + [P, A, E]
    toggle_off = np.zeros(E + 1, np.int32)
    ann_points = np.zeros(max(A, 1), np.int64)
    sizes = np.zeros(coco_masks.SIZES, np.int64)
    assert lib.tfb200_coco_poly_count_host(*geo, _p(toggle_off), _p(ann_points), _p(sizes)) == 0
    coco_masks.check_sizes(sizes, lambda: ann_points, names)
    run_off = np.zeros(A + 1, np.int64)
    runs = np.zeros((max(int(sizes[1]), 1), 2), np.uint32)
    assert lib.tfb200_coco_poly_runs_host(*geo, _p(toggle_off), int(sizes[1]), _p(run_off), _p(runs)) == 0
    return run_off, runs[:run_off[-1]].astype(np.int64), sizes


def host_list(lib, segs, hw):
    off, runs, _ = host_runs(lib, segs, hw)
    return [runs[off[a]:off[a + 1]] for a in range(len(segs))]


def check_against_oracle(lib, segs, h, w):
    got = host_list(lib, segs, [(h, w)] * len(segs))
    for seg, g in zip(segs, got):
        assert np.array_equal(g, ref.ann_runs(seg, h, w)), seg


# ---------------------------------------------------------------- the oracle on hand values

def test_oracle_square_and_box_list():
    counts = ref.fr_poly([0, 0, 10, 0, 10, 10, 0, 10], 20, 20)
    assert counts == [0] + [10, 10] * 9 + [10, 210]
    m = ref.decode(counts, 20, 20)
    assert m.sum() == 100 and m[:10, :10].all()
    assert np.array_equal(ref.ann_mask([[0, 0, 10, 10]], 20, 20), m)


def test_oracle_integer_rectangles_cover_w_times_h():
    rng = np.random.default_rng(0)
    for _ in range(50):
        x, y = (int(v) for v in rng.integers(0, 30, 2))
        bw, bh = (int(v) for v in rng.integers(1, 20, 2))
        m = ref.ann_mask([[x, y, x + bw, y, x + bw, y + bh, x, y + bh]], 50, 50)
        assert m.sum() == bw * bh and m[y:y + bh, x:x + bw].all()
        assert np.array_equal(ref.ann_mask([[x, y, bw, bh]], 50, 50), m)


def test_fma_hazard_example():
    """The issue's edge: ys = 2024, ye = -2692, dx = 9104, t = 3414."""
    s = (-2692 - 2024) / 9104
    assert ref._line(2024, s, 3414, False) == 256
    assert ref._line(2024, s, 3414, True) == 255


def fma_sensitive_edges(seed, count, h=1080, w=1920, budget=20000):
    """The exact search: long edges on the 5x grid where a fused ys + s * t + .5 changes a boundary point, kept when
    the triangle on the edge gets another mask."""
    rng = np.random.default_rng(seed)
    found = []
    for _ in range(budget):
        if len(found) == count:
            break
        dx = int(rng.integers(3000, 9000))
        ys = int(rng.integers(0, 5 * h))
        ye = ys + int(rng.integers(-min(dx, 5 * h), min(dx, 5 * h)))
        if ye < 0 or ye >= 5 * h:
            continue
        xs = int(rng.integers(0, 5 * w - dx))
        s = (ye - ys) / dx
        q = (ys + s * np.arange(dx + 1, dtype=np.float64)) + .5
        near = np.flatnonzero(np.abs(q - np.round(q)) < 1e-7).tolist()
        if not any(ref.c_int(float(Fraction(ys) + Fraction(s) * t) + .5) != ref.c_int(float(q[t])) for t in near):
            continue
        c = [pf.from_grid(v) for v in (xs, ys, xs + dx, ye)]
        poly = [c[0], c[1], c[2], c[3], c[0], c[3]]
        if ref.fr_poly(poly, h, w) != ref.fr_poly(poly, h, w, contract=True):
            found.append((xs, ys, xs + dx, ye))
    return found


def test_fma_edges_come_from_the_search_and_are_sensitive():
    assert fma_sensitive_edges(7, 2) == pf.FMA_EDGES[:2]
    for (xs, ys, xe, ye), seg in zip(pf.FMA_EDGES, pf.fma_polygons()):
        assert [ref.grid(c) for c in seg[0][:4]] == [xs, ys, xe, ye]
        assert not np.array_equal(ref.ann_mask(seg, 1080, 1920), ref.ann_mask(seg, 1080, 1920, contract=True))


# ---------------------------------------------------------------- the host build against the oracle

def test_host_build_hand_values(host_lib):
    square = [[0, 0, 10, 0, 10, 10, 0, 10]]
    (a, b), = [host_list(host_lib, [square, [[0, 0, 10, 10]]], [(20, 20)] * 2)]
    assert np.array_equal(a, np.stack((np.arange(10) * 20, np.full(10, 10)), 1))
    assert np.array_equal(a, b)


@pytest.mark.parametrize("seed,h,w", [(0, 23, 31), (1, 48, 64), (2, 97, 131), (3, 64, 48), (4, 1, 7), (5, 9, 1)])
def test_host_build_matches_oracle_random(host_lib, seed, h, w):
    check_against_oracle(host_lib, pf.segmentations(seed, 120, h, w), h, w)


def test_host_build_matches_oracle_overlapping_parts(host_lib):
    rng = np.random.default_rng(11)
    segs = []
    for _ in range(40):
        base = pf._part(rng, 60, 80, "star")
        shifted = [v + float(rng.integers(-6, 7)) for v in base]
        segs.append([base, shifted, pf._part(rng, 60, 80, "convex")])
    check_against_oracle(host_lib, segs, 60, 80)


def test_host_build_vertices_on_the_last_column_and_row(host_lib):
    h, w = 30, 40
    segs = [[[w - 1, 0, w - 1, h, 0, h, 0, 0]], [[0, h, w - 1, h, w - 1, 0]], [[w - 1.0, h, w, h + 1.0, w - 1, 3]],
            [[0, 0, w - 1, 0, w - 1, h - 1, 0, h - 1]], [[0.4, h - 0.6, w - 1.4, h, w - 1, 2.2]],
            [[w - 1, h, w - 1, h, w - 1, h]], [[-0.3, -0.1, -0.9, h + 0.3, w + 0.2, -0.7]]]
    check_against_oracle(host_lib, segs, h, w)


def test_host_build_fma_sensitive_edges(host_lib):
    check_against_oracle(host_lib, pf.fma_polygons(), 1080, 1920)


def test_host_build_rectangles_equal_rect_masks(host_lib):
    """Integer rectangle polygons are exactly the rect masks the evaluator cross-check uses."""
    rng = np.random.default_rng(4)
    boxes = [(int(x), int(y), int(x + bw), int(y + bh)) for x, y, bw, bh in
             zip(*[rng.integers(0, 40, 30) for _ in range(2)], *[rng.integers(1, 25, 30) for _ in range(2)])]
    segs = [[[x0, y0, x1, y0, x1, y1, x0, y1]] for x0, y0, x1, y1 in boxes]
    for (x0, y0, x1, y1), g in zip(boxes, host_list(host_lib, segs, [(64, 70)] * len(segs))):
        assert np.array_equal(g, ref.runs_of(ef.rect_mask((x0, y0, x1, y1), 64, 70)))


def test_host_rle_decode_and_mask_writer(host_lib):
    rng = np.random.default_rng(5)
    h, w = 17, 23
    masks = [rng.random((h, w)) < p for p in (0.0, 0.3, 0.7, 1.0)]
    strings = [mots.encode(m)["counts"] for m in masks] + [b"", b"1", b"0Y"]   # then malformed ones
    lens = np.asarray([len(s) for s in strings], np.int64)
    chars = np.frombuffer(b"".join(strings), np.uint8)
    str_off = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    cap_off = np.concatenate(([0], np.cumsum(lens // 2))).astype(np.int64)
    bounds = np.zeros((len(strings), 2), np.int64)
    runs = np.zeros((int(cap_off[-1]) + 1, 2), np.uint32)
    first_bad = np.asarray([len(strings)], np.int64)
    host_lib.tfb200_coco_rle_runs_host(_p(chars), _p(str_off), _p(cap_off), len(strings), h, w, _p(bounds),
                                       _p(runs), _p(first_bad))
    assert first_bad[0] == len(masks)
    for k, m in enumerate(masks):
        assert np.array_equal(runs[bounds[k, 0]:bounds[k, 1]].astype(np.int64), ref.runs_of(m))
    seg = [[1.5, 2, 20, 3.3, 11, 15.9]]
    off, pruns, _ = host_runs(host_lib, [seg], [(h, w)])
    src = np.asarray([-1, 0, -3, -2], np.int32)
    out = np.zeros((len(src), h, w), np.uint8)
    host_lib.tfb200_coco_masks_u8_host(_p(src), len(src), h, w, _p(off), _p(pruns.astype(np.uint32)), _p(bounds),
                                       _p(runs), _p(out))
    for o, want in zip(out, (masks[0], ref.ann_mask(seg, h, w), masks[2], masks[1])):
        assert np.array_equal(o, want.astype(np.uint8))


# ---------------------------------------------------------------- errors

@pytest.mark.parametrize("seg,match", [
    ([], "first part of at least 4"),
    ([[1, 2, 3]], "first part of at least 4"),
    ([[]], "first part of at least 4"),
    ([[0, 0, 4, 4], [1, 1, 2, 2, 3, 3]], "box-list segmentation has a part of 6"),
    ([[0, 0, 4, 0, float("nan"), 3]], "non-finite"),
    ([[0, 0, float("inf"), 0, 4, 3]], "non-finite"),
    ([[0, 0, 4.3e8, 0, 4, 3]], "overflows"),
    ([[0, 0, 4, 0, 4, -4.3e8]], "overflows"),
    ([[-4e8, 0, 4e8, 0, 0, 1]], "boundary points"),
])
def test_errors_name_the_annotation(host_lib, seg, match):
    good = [[1, 1, 5, 1, 5, 5]]
    with pytest.raises(ValueError, match=f"annotation 77.*{match}|annotation 77: .*{match}"):
        host_runs(host_lib, [good, seg, good], [(10, 10)] * 3, ["annotation 5", "annotation 77", "annotation 9"])


def test_points_over_the_limit_name_the_annotation_that_crosses_it(host_lib):
    long = [[-1e8, 0, 1e8, 0, 0, 1]]                      # about 2e9 points: two of them cross 2^31 - 1
    with pytest.raises(ValueError, match="annotation 2 takes the boundary points"):
        host_runs(host_lib, [[[1, 1, 5, 1, 5, 5]], long, long], [(10, 10)] * 3)


def test_ground_truth_without_device_rejects_polygons():
    ds = {"images": [{"id": 1, "height": 10, "width": 10}], "categories": [{"id": 1}],
          "annotations": [{"id": 3, "image_id": 1, "category_id": 1, "area": 16.0, "bbox": [1, 1, 4, 4],
                           "segmentation": [[1, 1, 5, 1, 5, 5, 1, 5]]}]}
    with pytest.raises(NotImplementedError, match="annotation 3"):
        coco_eval.GroundTruth(ds, True)
    coco_eval.GroundTruth(ds, False)                      # boxes alone never read the segmentation
