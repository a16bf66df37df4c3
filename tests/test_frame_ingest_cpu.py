"""Host side of the frame ingest (trackformer_b200/frame_ingest.py, csrc/frame_ingest.cu) without a GPU: the size rule,
Pillow's integer resampling restated in NumPy against bytes recorded from the reference's validation transform
(tests/golden/make_golden_frame_ingest.py) and against Pillow itself, the byte -> float table, the coefficient tables,
and argument validation of the C ABI, of FrameIngest and of Tracker.step."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR

BITS = 22


# ------------------------------------------------------------------------------------- the arithmetic, restated
def tables(n, m):
    """Pillow's bilinear coefficients for one axis of length n -> m, one output index at a time: (lo, cnt) [m, 2] and
    the weights quantised to 22 fractional bits [m, ksize]."""
    scale = n / m
    fs = max(scale, 1.0)
    support = fs
    ksize = int(math.ceil(support)) * 2 + 1
    bounds, kk = np.zeros((m, 2), np.int64), np.zeros((m, ksize), np.int64)
    for i in range(m):
        center = (i + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        cnt = min(int(center + support + 0.5), n) - lo
        w = [0.0] * ksize
        total = 0.0
        for j in range(cnt):
            a = abs((j + lo - center + 0.5) * (1.0 / fs))
            w[j] = 1.0 - a if a < 1.0 else 0.0
            total += w[j]
        for j in range(cnt):
            if total != 0.0:
                w[j] /= total
        kk[i] = [int(0.5 + v * (1 << BITS)) for v in w]
        bounds[i] = lo, cnt
    return bounds, kk


def pass1d(img, m):
    """one pass along axis 1 of uint8 [A, n, C]: 32-bit accumulator, rounded and clamped to a byte"""
    bounds, kk = tables(img.shape[1], m)
    out = np.empty((img.shape[0], m, img.shape[2]), np.uint8)
    src = img.astype(np.int64)
    for i in range(m):
        lo, cnt = bounds[i]
        acc = (1 << (BITS - 1)) + np.tensordot(src[:, lo:lo + cnt, :], kk[i, :cnt], axes=([1], [0]))
        assert acc.max() < 2 ** 31
        out[:, i, :] = np.clip(acc >> BITS, 0, 255).astype(np.uint8)
    return out


def resize_u8(img, oh, ow):
    """horizontal pass, then vertical, each skipped when its length stays"""
    h, w, _ = img.shape
    x = img
    if ow != w:
        x = pass1d(x, ow)
    if oh != h:
        x = pass1d(x.transpose(1, 0, 2), oh).transpose(1, 0, 2)
    return x


def restated_img(frame, val_width=800, max_size=1333):
    """uint8 [H, W, 3] -> fp32 [1, 3, h, w], what the ingest must return (host restatement)"""
    from trackformer_b200.frame_ingest import normalise_table, val_size
    h, w = val_size(frame.shape[0], frame.shape[1], val_width, max_size)
    resized = torch.from_numpy(resize_u8(frame, h, w)).long()
    lut = normalise_table()
    return torch.stack([lut[c][resized[:, :, c]] for c in range(3)])[None]


def synthetic_frame(h, w, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    img[: h // 4] = np.where(rng.random((h // 4, w, 1)) > 0.5, 255, 0)
    img[h // 4: h // 2, :, 1] = (np.arange(w) * 255 // max(w - 1, 1)).astype(np.uint8)[None, :]
    return img


def golden():
    with np.load(os.path.join(GOLDEN_DIR, "frame_ingest.npz")) as z:
        data = {k: z[k] for k in z.files}
    return [str(n) for n in data["names"]], data


NAMES, GOLD = golden()


# ------------------------------------------------------------------------------------------------------ val_size
def test_fixture_covers_the_cases_it_should():
    kinds = set()
    for n in NAMES:
        (H, W), (h, w) = GOLD[f"{n}_orig_size"], GOLD[f"{n}_size"]
        val_width, max_size = GOLD[f"{n}_settings"]
        kinds.add("down" if h < H else "up" if h > H else "same")
        kinds.add("landscape" if W > H else "portrait")
        if min(h, w) != val_width:
            kinds.add("capped")
        if H % 2 and W % 2:
            kinds.add("odd")
    assert kinds >= {"down", "up", "same", "landscape", "portrait", "capped", "odd"}


@pytest.mark.parametrize("name", NAMES)
def test_val_size_equals_recorded(name):
    from trackformer_b200.frame_ingest import val_size
    H, W = (int(v) for v in GOLD[f"{name}_orig_size"])
    val_width, max_size = (int(v) for v in GOLD[f"{name}_settings"])
    assert val_size(H, W, val_width, max_size) == tuple(int(v) for v in GOLD[f"{name}_size"])


@pytest.mark.parametrize("shape,want", [
    ((1080, 1920), (750, 1333)),          # capped: round(1333 * 1080 / 1920) = 750, int(750 * 1920 / 1080) = 1333
    ((480, 640), (800, 1066)),            # int(800 * 640 / 480) = 1066 (1066.67 truncated)
    ((1333, 800), (1333, 800)),           # portrait already at the target
    ((800, 1333), (800, 1333)),
    ((1920, 1080), (1333, 750)),
    ((600, 1001), (799, 1332)),           # round gives 799.0 -> 799, then 799 * 1001 / 600 = 1332.998 truncates to 1332
    ((500, 500), (800, 800)),
])
def test_val_size_hand_worked(shape, want):
    from trackformer_b200.frame_ingest import val_size
    assert val_size(*shape) == want


def test_val_size_rejects_nonsense():
    from trackformer_b200.frame_ingest import val_size
    with pytest.raises(ValueError):
        val_size(0, 10)
    with pytest.raises(ValueError):
        val_size(10, 10, val_width=0)


# ---------------------------------------------------------------------------------------------------- resampling
@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_reference_bytes(name):
    h, w = (int(v) for v in GOLD[f"{name}_size"])
    got = resize_u8(GOLD[f"{name}_frame"], h, w)
    np.testing.assert_array_equal(got, GOLD[f"{name}_resized"])


@pytest.mark.parametrize("name", NAMES)
def test_restated_image_equals_reference_float(name):
    val_width, max_size = (int(v) for v in GOLD[f"{name}_settings"])
    got = restated_img(GOLD[f"{name}_frame"], val_width, max_size)
    assert torch.equal(got[0], torch.from_numpy(GOLD[f"{name}_img"]))


@pytest.mark.parametrize("shape,out", [((1080, 1920), (750, 1333)), ((480, 640), (800, 1066)),
                                       ((270, 1920), (50, 1920))])
def test_restatement_equals_pillow(shape, out):
    Image = pytest.importorskip("PIL.Image")
    frame = synthetic_frame(*shape, seed=3)
    want = np.asarray(Image.fromarray(frame).resize((out[1], out[0]), Image.BILINEAR))
    np.testing.assert_array_equal(resize_u8(frame, *out), want)


@pytest.mark.parametrize("n,m", [(1920, 1333), (1080, 750), (640, 1066), (480, 800), (1080, 200), (517, 51), (5, 9),
                                 (7, 12), (403, 40), (3000, 7)])
def test_coefficient_tables(n, m):
    from trackformer_b200.frame_ingest import resample_table
    table = resample_table(n, m)
    bounds, kk = tables(n, m)
    ksize = kk.shape[1]
    assert table.dtype == np.int32 and table.shape == (m, 2 + ksize)
    np.testing.assert_array_equal(table[:, :2], bounds)
    np.testing.assert_array_equal(table[:, 2:], kk)
    lo, cnt = table[:, 0].astype(np.int64), table[:, 1].astype(np.int64)
    assert (lo >= 0).all() and (cnt >= 1).all() and (cnt <= ksize).all() and (lo + cnt <= n).all()
    assert (np.diff(lo) >= 0).all()
    assert (np.abs(table[:, 2:].astype(np.int64).sum(1) - (1 << BITS)) <= ksize).all()
    assert (table[:, 2:] >= 0).all()
    for i in range(m):
        assert not table[i, 2 + cnt[i]:].any()


def test_normalise_table_equals_to_tensor_and_normalize():
    from trackformer_b200.frame_ingest import normalise_table
    lut = normalise_table()
    assert lut.dtype == torch.float32 and tuple(lut.shape) == (3, 256)
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    u = torch.arange(256, dtype=torch.uint8).view(1, 256, 1).expand(3, 256, 1).contiguous()
    want = u.float().div(255)
    want = want.sub(torch.tensor(mean).view(3, 1, 1)).div(torch.tensor(std).view(3, 1, 1))
    assert torch.equal(lut, want[:, :, 0])
    tvf = pytest.importorskip("torchvision.transforms.functional")
    Image = pytest.importorskip("PIL.Image")
    pil = Image.fromarray(np.arange(256, dtype=np.uint8).reshape(256, 1, 1).repeat(3, 2))
    assert torch.equal(lut, tvf.normalize(tvf.to_tensor(pil), mean, std)[:, :, 0])


# ---------------------------------------------------------------------------------------------------- validation
def test_abi_argument_validation_without_gpu():
    from trackformer_b200 import _build
    lib = ctypes.CDLL(_build.build_library())
    f = lib.tfb200_frame_ingest_u8_f32
    vp, i, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    f.restype = i
    f.argtypes = [vp, i64, i, i, vp, i, i, vp, i, i, vp, vp, i64, i64, i, i, vp]
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, vp)

    def call(src=p, stride=3 * 20, H=10, W=20, xtab=p, ksx=5, cx=5, ytab=p, ksy=5, cy=4, lut=p, dst=p, drow=16,
             dplane=160, h=8, w=16):
        return f(src, stride, H, W, xtab, ksx, cx, ytab, ksy, cy, lut, dst, drow, dplane, h, w, None)
    assert call(src=None) == -1 and call(lut=None) == -1 and call(dst=None) == -1
    assert call(H=0) == -2 and call(W=-1) == -2 and call(h=0) == -2 and call(w=0) == -2
    assert call(stride=3 * 20 - 1) == -2                   # rows overlap
    assert call(drow=15) == -2
    assert call(cx=6) == -2 and call(cy=6) == -2           # cnt > ksize
    assert call(ksx=0, cx=0) == -2
    assert call(xtab=None) == -2                           # no table although the width changes
    assert call(ytab=None) == -2


def test_check_frame_names_the_layout():
    from trackformer_b200.frame_ingest import check_frame
    assert check_frame(np.zeros((4, 5, 3), np.uint8)) == ("numpy", 4, 5)
    assert check_frame(torch.zeros(4, 5, 3, dtype=torch.uint8)) == ("cpu", 4, 5)
    assert check_frame(np.zeros((8, 5, 3), np.uint8)[::2]) == ("numpy", 4, 5)       # host frames may be strided
    for bad in (np.zeros((4, 5, 3), np.float32), torch.zeros(3, 4, 5, dtype=torch.uint8),
                np.zeros((4, 5, 4), np.uint8), torch.zeros(1, 4, 5, 3, dtype=torch.uint8),
                torch.zeros(4, 5, 3), [[0, 0, 0]], np.zeros((0, 5, 3), np.uint8)):
        with pytest.raises(ValueError, match=r"\[H, W, 3\]"):
            check_frame(bad)


def test_frame_ingest_constructor_validation():
    from trackformer_b200.frame_ingest import FrameIngest
    with pytest.raises(RuntimeError, match="no CPU path"):
        FrameIngest("cpu")
    with pytest.raises(ValueError):
        FrameIngest("cuda", val_width=0)
    with pytest.raises(ValueError):
        FrameIngest("cuda", max_size=-5)
    with pytest.raises(ValueError):
        FrameIngest("cuda", mean=(0.5, 0.5))
    with pytest.raises(ValueError):
        FrameIngest("cuda", std=(0.2, 0.0, 0.2))


@pytest.mark.parametrize("tracker", ["Tracker", "DeviceTracker"])
def test_step_rejects_img_and_frame_together(tracker):
    import tracker_fixtures as tf
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.tracker import Tracker
    cls = {"Tracker": Tracker, "DeviceTracker": DeviceTracker}[tracker]
    det = tf.ScriptedDetector(tf.Scene(seed=0), overflow_boxes=False)
    tr = cls(det, {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), False)
    assert tr.frame_ingest is None
    tr.reset()
    blob = next(iter(tf.blobs(tf.Scene(seed=0), 1)))
    blob["frame"] = np.zeros((tf.IMG_H, tf.IMG_W, 3), np.uint8)
    with pytest.raises(ValueError, match='both "img" and "frame"'):
        tr.step(blob)
    assert tr.frame_index == 0
    given = object()
    assert cls(det, {"bbox": DeformablePostProcess()}, tf.tracker_cfg("default"), frame_ingest=given).frame_ingest is given
