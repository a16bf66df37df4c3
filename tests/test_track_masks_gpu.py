"""Tracking with segmentation masks on the GPU: csrc/track_masks.cu against the torch composition and a fp64
recomputation, the row-selective mask head on CUDA, and Tracker / DeviceTracker with masks against the label maps
recorded from the reference (tests/golden/make_golden_track_masks.py)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import track_mask_fixtures as tmf
import tracker_fixtures as tf
from test_track_masks_cpu import check_masks_against_gold
from test_tracker_cpu import check_against_gold

pytestmark = pytest.mark.gpu

EPS = 1e-5          # probability band around a decision inside which fp32 rounding order may decide a pixel
DEEP = 1 - 1e-9     # fp64 values above this are exactly 1.0 in any fp32 evaluation: ties there must be resolved exactly


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def oracle(logits, src, ids, prev, size, crop, orig):
    """(label of the CPU torch composition, pixels a fp64 recomputation puts within EPS of a decision)"""
    from trackformer_b200.segmentation import resolve_track_masks
    logits = logits.cpu()
    prev = None if prev is None else prev.cpu()
    want = resolve_track_masks(logits, src, ids, prev, size, crop, orig)
    H, W = orig
    src_t = torch.as_tensor(src).long()
    vals = torch.zeros(len(src), H, W, dtype=torch.float64)
    fresh = src_t >= 0
    if fresh.any():
        p = F.interpolate(logits.double()[src_t[fresh]][None], size=tuple(size), mode="bilinear",
                          align_corners=False).sigmoid()[0, :, :crop[0], :crop[1]]
        vals[fresh] = F.interpolate(p[:, None], size=(H, W), mode="nearest")[:, 0]
    for t in torch.nonzero(~fresh).flatten().tolist():
        vals[t] = (prev == int(ids[t])).double()
    if len(src) == 0:
        return want, torch.zeros(H, W, dtype=torch.bool)
    top = vals.topk(min(2, len(src)), 0).values
    near = (top[0] - 0.5).abs() < EPS
    if len(src) > 1:
        gap = top[0] - top[1]
        near |= (gap > 0) & (gap < EPS) & ~(top[1] >= DEEP)
    return want, near


def run_case(dev, T, h, w, size, crop, orig, stale=0, seed=0, zero=False, ties=False, cap=0.05):
    """random logits (x4: many saturated values, so a few % of the pixels of 150 tracks sit in the EPS band)"""
    from trackformer_b200.segmentation import resolve_track_masks
    g = torch.Generator().manual_seed(seed)
    K = T - stale
    logits = torch.randn(K, h, w, generator=g) * 4
    if zero:
        logits.zero_()
    if ties and K >= 2:                                  # saturated blocks overlapping across rows: exact fp32 ties
        for k in range(K):
            y0, x0 = int(torch.randint(0, h // 2, (1,), generator=g)), int(torch.randint(0, w // 2, (1,), generator=g))
            logits[k, y0:y0 + h // 2, x0:x0 + w // 2] = 30.0 + 10.0 * (k % 3)
    ids = (torch.randperm(4 * T + 8, generator=g)[:T] * 3 + 2).int()
    order = torch.randperm(T, generator=g)
    src = torch.full((T,), -1, dtype=torch.int32)
    src[order[:K]] = torch.arange(K, dtype=torch.int32)
    prev = None
    if stale:
        pool = torch.cat([ids, torch.tensor([-1, 999999], dtype=torch.int32)])      # fresh ids and unknown ids too
        blocks = pool[torch.randint(0, len(pool), (8, 8), generator=g)]
        prev = F.interpolate(blocks[None, None].float(), size=tuple(orig), mode="nearest")[0, 0].int()
    got = resolve_track_masks(logits.to(dev), src, ids, None if prev is None else prev.to(dev), size, crop, orig)
    assert got.is_cuda and got.dtype == torch.int32 and tuple(got.shape) == tuple(orig)
    want, near = oracle(logits, src.tolist(), ids.tolist(), prev, size, crop, orig)
    diff = got.cpu() != want
    assert not (diff & ~near).any(), f"{int((diff & ~near).sum())} pixels differ outside the EPS band"
    assert near.float().mean() <= cap
    return got.cpu(), want


@pytest.mark.parametrize("T,h,w,size,crop,orig,stale", [
    (150, 27, 37, (118, 157), (118, 157), (480, 640), 20),     # non-integer scales, orig larger than size
    (1, 20, 30, (80, 120), (70, 100), (50, 70), 0),            # crop smaller than size, orig smaller than the crop
    (5, 16, 16, (64, 64), (64, 64), (128, 128), 2),            # identity-free 4x bilinear, exact 2x nearest
    (3, 33, 41, (33, 41), (33, 41), (33, 41), 1),              # identity everywhere
    (7, 200, 300, (800, 1200), (800, 1200), (40, 60), 0),      # footprint beyond the shared-memory stage
    (300, 12, 14, (45, 50), (45, 50), (90, 140), 100),         # several chunks of tracks
])
def test_kernel_matches_oracle(dev, T, h, w, size, crop, orig, stale):
    run_case(dev, T, h, w, size, crop, orig, stale=stale)


def test_kernel_exact_ties_and_stale(dev):
    got, want = run_case(dev, 12, 24, 32, (96, 128), (96, 128), (192, 256), stale=4, ties=True, seed=3)
    assert (got >= 0).any()
    got, want = run_case(dev, 12, 24, 32, (96, 128), (96, 128), (192, 256), stale=0, ties=True, seed=4)


def test_kernel_all_stale_zero_logits_and_empty(dev):
    from trackformer_b200.segmentation import resolve_track_masks
    got, _ = run_case(dev, 6, 10, 10, (40, 40), (40, 40), (64, 96), stale=6, seed=5)
    assert (got >= 0).any()
    got, _ = run_case(dev, 4, 10, 12, (40, 48), (40, 48), (80, 96), zero=True, cap=1.0)
    assert (got == -1).all()                              # sigmoid(0) = 0.5 is not foreground
    empty = resolve_track_masks(torch.zeros(0, 4, 4, device=dev), [], [], None, (8, 8), (8, 8), (16, 16))
    assert empty.is_cuda and (empty == -1).all()


@pytest.mark.parametrize("case", list(tf.CASES))
@pytest.mark.parametrize("tracker", ["Tracker", "DeviceTracker"])
def test_trackers_with_masks_on_cuda_match_reference(dev, case, tracker):
    """scripted masks on the GPU: same decisions as the reference, label maps equal except inside the EPS band"""
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.segmentation import PostProcessSegm
    from trackformer_b200.tracker import Tracker
    import trackformer_b200.tracker as tmod
    calls = []
    real = tmod.resolve_track_masks

    def recording(logits, src, ids, prev, size, crop, orig):
        calls.append((logits.detach().cpu().clone(), list(src), list(ids), None if prev is None else prev.cpu().clone(),
                      tuple(size), tuple(crop), tuple(orig)))
        return real(logits, src, ids, prev, size, crop, orig)
    tmod.resolve_track_masks = recording
    try:
        cls = {"Tracker": Tracker, "DeviceTracker": DeviceTracker}[tracker]
        out = tmf.run_case(cls, DeformablePostProcess(), PostProcessSegm(), case, device=dev)
    finally:
        tmod.resolve_track_masks = real
    check_against_gold({k: v for k, v in out.items() if k != "labels"}, case, rtol=1e-5)
    frames = sorted(set(out["rows"][:, 1].astype(int).tolist()))     # frames without results make no call
    assert len(frames) == len(calls)
    band = np.zeros_like(out["labels"], dtype=bool)
    for f, c in zip(frames, calls):
        band[f] = oracle(*c)[1].numpy()
    check_masks_against_gold(out, f"tracker_masks_{case}", lambda g: band)


@pytest.mark.parametrize("k,bucket", [(0, 16), (21, 32)])
def test_row_selective_head_on_cuda(dev, k, bucket):
    """mask_logits(rows) -- model and GraphedDetector (graph replay) -- against the full forward's pred_masks rows"""
    import model_fixtures as mf
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args
    torch.manual_seed(0)
    model, _, _ = build_model(default_args(True, False, device=str(dev), masks=True))
    mf.canonical_weights_(model, 0)
    model.to(dev)
    model.tracking()
    prev_tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        f1, f2 = (f.to(dev) for f in tf.model_frames((160, 224), 2))
        with torch.no_grad():
            o1, _, feat1, _, _ = model(f1[None], None, None)
            tgt = None
            if k:
                tgt = [{"track_query_boxes": o1["pred_boxes"][0, :k].clone(),
                        "track_query_hs_embeds": o1["hs_embed"][0, :k].clone(), "image_id": torch.tensor([1], device=dev)}]
            full, _, _, _, _ = model(f2[None], tgt, feat1)
            rows = [0, k + 5, k + model.num_queries - 1] + ([k - 1, 2] if k > 2 else [])
            _, _, feats, mem, hs = model.detect(f2[None], tgt, feat1)
            sel = model.mask_logits(feats, mem, hs, rows)
            det = GraphedDetector(model, bucket=bucket)
            for _ in range(2):
                out, *_ = det.detect(f2[None], tgt, feat1)
                g = det.mask_logits(rows)
        want = full["pred_masks"][:, rows]
        assert "pred_masks" not in out and det.replays == 2
        torch.testing.assert_close(sel, want, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(g, want, rtol=1e-3, atol=1e-3)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev_tf32


def test_graphed_tracker_with_masks_equals_padded_eager(dev):
    """Tracker + GraphedDetector with masks: the graphed and the padded eager program take the same decisions and
    produce the same label maps (same kernels on the same inputs), on the real segmentation model"""
    from trackformer_b200.deformable_detr import DeformablePostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.segmentation import PostProcessSegm
    from trackformer_b200.tracker import Tracker

    def build(tracking, multi_frame, **overrides):
        torch.manual_seed(0)
        model, criterion, _ = build_model(default_args(tracking, multi_frame, device=str(dev), **overrides))
        return model, criterion
    cfg = dict(detection_obj_score_thresh=0.3, track_obj_score_thresh=0.3, reid_score_thresh=0.3,
               inactive_patience=3, reid_sim_threshold=2.0, detection_nms_thresh=0.7, track_nms_thresh=0.7,
               steps_termination=2)
    outs = {}
    for name, cls, graphs in (("graph", Tracker, True), ("padded", Tracker, False), ("device", DeviceTracker, True)):
        outs[name] = tmf.run_model_sequence(build, cls, DeformablePostProcess(), PostProcessSegm(), cfg, device=dev,
                                            n_frames=4, out_lay_scale=8.0,
                                            wrap=lambda m, g=graphs: GraphedDetector(m, bucket=16, use_graphs=g))
    a = outs["graph"]
    assert len(a["rows"]) > 0 and (a["labels"] >= 0).any()
    for other in ("padded", "device"):
        b = outs[other]
        for key in ("num_reids", "track_num", "active_ids", "inactive_ids"):
            np.testing.assert_array_equal(a[key], b[key], err_msg=f"{other}: {key}")
        np.testing.assert_array_equal(a["rows"][:, :3], b["rows"][:, :3])
        mismatch = float((a["labels"] != b["labels"]).mean())
        assert mismatch < 1e-4, f"{other}: {mismatch:.2e} of the pixels differ"
