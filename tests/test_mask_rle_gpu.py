"""COCO run-length encodings on the GPU: csrc/mask_rle.cu byte for byte against trackformer_b200.mots.encode on
resolved label maps, rectangles, edge cases and the worst case, and Tracker / DeviceTracker with mask_rle=True against
their bool masks on the scripted scenes and the seeded segmentation model."""
import numpy as np
import pytest
import torch

import tracker_fixtures as tf
from test_mask_rle_cpu import _run_scripted, check_rle_results
from trackformer_b200.mots import encode, label_map_rle, write_results

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def check(dev, lab, ids):
    """the kernel's RLEs of a host label map == encode of each mask; returns them"""
    lab = np.asarray(lab, np.int32)
    got = label_map_rle(torch.from_numpy(lab).to(dev), ids)
    flat = np.ascontiguousarray(lab.T)
    for t, i in enumerate(ids):
        want = encode((flat == i).T)
        assert got[t] == want, f"track {t} (id {i}): {got[t]['counts'][:40]!r} != {want['counts'][:40]!r}"
    return got


def resolved_map(dev, T, H, W, seed):
    """resolve_track_masks (csrc/track_masks.cu) of random stride-4 logits: many short runs per column"""
    from trackformer_b200.segmentation import resolve_track_masks
    g = torch.Generator().manual_seed(seed)
    size = ((H + 3) // 4 * 4, (W + 3) // 4 * 4)
    logits = torch.randn(T, size[0] // 4, size[1] // 4, generator=g) * 4
    ids = (torch.randperm(4 * T + 8, generator=g)[:T] * 7 + 3).int()
    lab = resolve_track_masks(logits.to(dev), list(range(T)), ids.tolist(), None, size, size, (H, W))
    return lab, ids.tolist()


@pytest.mark.parametrize("H,W", [(800, 1333), (1080, 1920)])
@pytest.mark.parametrize("T", [1, 37, 150, 300])
def test_kernel_on_resolved_label_maps(dev, H, W, T):
    lab, ids = resolved_map(dev, T, H, W, seed=T)
    host = lab.cpu().numpy()
    assert (host >= 0).any()
    check(dev, host, ids + [1])                           # plus an id that is not on the map


@pytest.mark.parametrize("H,W,T", [(800, 1333, 100), (1080, 1920, 100), (37, 29, 5)])
def test_kernel_on_rectangles(dev, H, W, T):
    rng = np.random.default_rng(T + H)
    lab = np.full((H, W), -1, np.int32)
    ids = [int(v) for v in rng.permutation(10 * T)[:T]]
    for i in ids:                                         # person-like boxes, later ones on top
        h, w = int(rng.integers(1, H // 2 + 1)), int(rng.integers(1, W // 4 + 1))
        y, x = int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1))
        lab[y:y + h, x:x + w] = i
    lab[0, :] = ids[0]                                    # runs across every column boundary
    lab[-1, -1] = ids[1]                                  # the last pixel
    check(dev, lab, ids)


def test_kernel_edge_cases(dev):
    rng = np.random.default_rng(5)
    lab = rng.integers(-3, 4, (61, 47)).astype(np.int32)
    lab[10:20, 5:9] = (1 << 30) + 1
    lab[30:, 40:] = (1 << 31) - 1
    ids = [0, 2, 9, (1 << 30) + 1, (1 << 31) - 1, 12345, 2]      # empty masks, absent ids, a repeated id
    check(dev, lab, ids)
    check(dev, np.full((13, 11), 7, np.int32), [7, 8])            # a full mask and an empty one
    for shape in ((1, 257), (257, 1), (1, 1), (1, 2)):             # a single row, a single column, one pixel
        check(dev, rng.integers(-1, 3, shape).astype(np.int32), [0, 1, 2])
    assert label_map_rle(torch.zeros(4, 5, dtype=torch.int32, device=dev), []) == []
    with pytest.raises(ValueError):
        label_map_rle(torch.zeros(4, 5, dtype=torch.int32, device=dev), [1, -2])


@pytest.mark.parametrize("H,W", [(1080, 1920), (33, 17)])
def test_kernel_worst_case_checkerboard(dev, H, W):
    """every pixel differs from the one before it in column-major order, so each ends one run and starts another: the
    largest boundary list and string the buffers must hold"""
    y, x = np.mgrid[:H, :W]
    lab = np.where((x * H + y) % 2 == 0, 5, 1 << 29).astype(np.int32)
    got = check(dev, lab, [5, 1 << 29])
    assert min(len(r["counts"]) for r in got) >= H * W                 # H * W or H * W + 1 counts of one character


def test_kernel_salt_and_pepper_and_repeat_calls(dev):
    rng = np.random.default_rng(7)
    lab = rng.integers(-1, 200, (512, 700)).astype(np.int32)
    ids = [int(v) for v in rng.permutation(220)[:150]]
    first = check(dev, lab, ids)
    d = torch.from_numpy(lab).to(dev)
    for _ in range(2):
        assert label_map_rle(d, ids) == first               # byte-identical run to run


@pytest.mark.parametrize("case", list(tf.CASES))
@pytest.mark.parametrize("tracker", ["Tracker", "DeviceTracker"])
def test_trackers_mask_rle_on_cuda(dev, case, tracker, tmp_path):
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.tracker import Tracker
    cls = {"Tracker": Tracker, "DeviceTracker": DeviceTracker}[tracker]
    plain = _run_scripted(cls, case, False, device=dev)
    rle = _run_scripted(cls, case, True, device=dev)
    assert check_rle_results(plain.results, rle.results) > 0
    fa = write_results(plain.results, str(tmp_path / "a"), "seq")
    fb = write_results(rle.results, str(tmp_path / "b"), "seq")
    assert open(fa, "rb").read() == open(fb, "rb").read()


@pytest.mark.parametrize("tracker", ["Tracker", "DeviceTracker"])
def test_trackers_mask_rle_on_segmentation_model(dev, tracker, tmp_path):
    """the seeded segmentation model over the CUDA-graph detector (tmf.run_model_sequence's set-up): the RLE results
    are the bool results' encodings, and the result files are equal"""
    import model_fixtures as mf
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.segmentation import PostProcessSegm
    from trackformer_b200.tracker import Tracker
    torch.manual_seed(0)
    model, _, _ = build_model(default_args(True, False, device=str(dev), masks=True))
    mf.canonical_weights_(model, 0)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "class_embed" in name and name.endswith("bias"):
                p[0] += 6.0
        model.mask_head.out_lay.weight.mul_(8.0)
        model.mask_head.out_lay.bias.mul_(8.0)
    model.to(dev)
    model.tracking()
    cfg = dict(tf.BASE_CFG)
    cfg.update(detection_obj_score_thresh=0.3, track_obj_score_thresh=0.3, reid_score_thresh=0.3, inactive_patience=3,
               reid_sim_threshold=2.0, detection_nms_thresh=0.7, track_nms_thresh=0.7, steps_termination=2)
    cls = {"Tracker": Tracker, "DeviceTracker": DeviceTracker}[tracker]
    size = (128, 160)
    orig = torch.tensor([[size[0] * 4, size[1] * 4]])
    runs = []
    for rle in (False, True):
        tr = cls(GraphedDetector(model, bucket=16), {"bbox": DeformablePostProcess(), "segm": PostProcessSegm()}, cfg,
                 False, mask_rle=rle)
        tr.reset()
        with torch.no_grad():
            for frame in tf.model_frames(size, 4):
                tr.step({"img": frame[None], "orig_size": orig, "dets": torch.zeros(1, 0, 4),
                         "size": torch.tensor([list(size)])})
        runs.append(tr.results)
    assert check_rle_results(*runs) > 0
    assert any(np.asarray(r["mask"]).any() for t in runs[0].values() for r in t.values())
    fa = write_results(runs[0], str(tmp_path / "a"), "seq")
    fb = write_results(runs[1], str(tmp_path / "b"), "seq")
    assert open(fa, "rb").read() == open(fb, "rb").read()
