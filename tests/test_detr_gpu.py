"""The vanilla-DETR family on the H100 kernels (dense attention, small attention, fused FFN / norms, mask head) against
fixtures recorded from the reference's own classes (tests/golden/make_golden_detr.py), the softmax post-processing
kernel against PostProcess, GraphedDetector / Tracker / DeviceTracker with DETRSegmTracking, and the graphed TrainStep
against the eager one for vanilla detection."""
import copy

import numpy as np
import pytest
import torch

import detr_fixtures as df
import track_mask_fixtures as tmf
from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture()
def strict_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.fixture()
def tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _worst(res, gold, keys):
    return {k: float(np.abs(np.asarray(res[k]) - gold[k]).max() / (np.abs(gold[k]).max() or 1.0)) for k in keys}


@pytest.mark.parametrize("case", ["det_mini", "det_padded_batch", "det_800x1333", "track_two_frames", "track_800x1333",
                                  "segm_track_two_frames"])
def test_forward_matches_reference_fp32(cuda_device, strict_fp32, case):
    df.check(df.run_case(case, cuda_device), load_golden(case, "detr_"), rtol=1e-3, rel_atol=1e-3)


@pytest.mark.parametrize("case,keys", [("det_800x1333", ["pred_logits", "pred_boxes"]),
                                       ("track_800x1333", ["f1_logits", "f1_boxes", "f2_logits", "f2_boxes"])])
def test_forward_matches_reference_tf32(cuda_device, tf32, case, keys):
    gold = load_golden(case, "detr_")
    res = df.run_case(case, cuda_device)
    print("tf32", _worst(res, gold, keys))
    df.check({k: res[k] for k in keys}, {k: gold[k] for k in keys}, rtol=1e-3, rel_atol=1e-3)


@pytest.mark.parametrize("case", ["train_step_det", "train_step_tracking", "segm_det_mini"])
def test_eager_train_step_matches_reference(cuda_device, strict_fp32, case):
    """The eager composition (model + criterion + backward): detection, the tracking route (non-focal criteria run
    eagerly) and the segmentation model with its mask losses."""
    gold = load_golden(case, "detr_")
    df.check(df.run_case(case, cuda_device), gold, rtol=5e-3, rel_atol=2e-3)


def test_packed_kernel_matches_postprocess(cuda_device):
    from trackformer_b200.deformable_detr import PostProcess
    gold = load_golden("postprocess", "detr_")
    g = torch.Generator().manual_seed(4)
    cases = [(torch.from_numpy(gold["logits"]), torch.from_numpy(gold["boxes"]), torch.from_numpy(gold["sizes"])),
             (torch.randn(1, 400, 92, generator=g) * 4, torch.rand(1, 400, 4, generator=g), torch.tensor([[1080, 1920]]))]
    for logits, boxes, sizes in cases:
        outputs = {"pred_logits": logits.to(cuda_device), "pred_boxes": boxes.to(cuda_device)}
        rows = PostProcess().packed(outputs, sizes.to(cuda_device))
        ref = PostProcess()(outputs, sizes.to(cuda_device))
        for i, r in enumerate(ref):
            torch.testing.assert_close(rows[i, :, 0], r["scores"], rtol=2e-6, atol=1e-7)
            assert torch.equal(rows._labels[i], r["labels"]) and torch.equal(rows[i, :, 1], r["labels"].float())
            torch.testing.assert_close(rows[i, :, 2:], r["boxes"], rtol=1e-6, atol=1e-3)
    assert int(PostProcess().packed({"pred_logits": cases[0][0].to(cuda_device), "pred_boxes": cases[0][1].to(cuda_device)},
                                    cases[0][2].to(cuda_device))._labels[0, 3]) == 2          # tie -> smaller class


def _track_cfg():
    return dict(detection_obj_score_thresh=0.3, track_obj_score_thresh=0.3, reid_score_thresh=0.3, inactive_patience=3,
                reid_sim_threshold=2.0, detection_nms_thresh=0.7, track_nms_thresh=0.7, steps_termination=2)


def test_trackers_with_masks_graphed_eager_and_device_agree(cuda_device, strict_fp32):
    """DETRSegmTracking through Tracker (eager model, GraphedDetector replay, padded eager) and DeviceTracker (graph
    replay), with the softmax PostProcess and masks: the same decisions and label maps."""
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.segmentation import PostProcessSegm
    from trackformer_b200.tracker import Tracker

    def build(tracking, multi_frame, **kw):
        return df.build(tracking, multi_frame, device=str(cuda_device), dataset="mot", **kw)
    outs = {}
    arms = (("eager", Tracker, None), ("graph", Tracker, True), ("padded", Tracker, False),
            ("device", DeviceTracker, True))
    for name, cls, graphs in arms:
        wrap = None if graphs is None else (lambda m, g=graphs: GraphedDetector(m, bucket=16, use_graphs=g))
        outs[name] = tmf.run_model_sequence(build, cls, PostProcess(), PostProcessSegm(), _track_cfg(), device=cuda_device,
                                            n_frames=5, out_lay_scale=8.0, wrap=wrap)
    a = outs["graph"]
    assert len(a["rows"]) > 0 and (a["labels"] >= 0).any() and int(a["track_num"]) > 0
    for other in ("eager", "padded", "device"):
        b = outs[other]
        for key in ("num_reids", "track_num", "active_ids", "inactive_ids"):
            np.testing.assert_array_equal(a[key], b[key], err_msg=f"{other}: {key}")
        np.testing.assert_array_equal(a["rows"][:, :3], b["rows"][:, :3])
        np.testing.assert_allclose(a["rows"], b["rows"], rtol=1e-4, atol=1e-3, err_msg=other)
        mismatch = float((a["labels"] != b["labels"]).mean())
        assert mismatch < 1e-4, f"{other}: {mismatch:.2e} of the pixels differ"


def test_graphed_detector_equals_eager_with_changing_track_counts(cuda_device, strict_fp32):
    from trackformer_b200.graphed_detector import GraphedDetector
    model, _ = df.build(True, False, device=str(cuda_device))
    import model_fixtures as mf
    mf.canonical_weights_(model, 0)
    model.to(cuda_device).tracking()
    graphed = GraphedDetector(model, bucket=8)
    frames = mf.make_images(7, [(160, 224)] * 5, cuda_device)
    prev = None
    with torch.no_grad():
        for i, (f, k) in enumerate(zip(frames, (0, 5, 12, 3, 12))):
            tgt = None
            if k:
                tgt = [{"track_query_boxes": prev["pred_boxes"][0, :k], "track_query_hs_embeds": prev["hs_embed"][0, :k],
                        "image_id": torch.tensor([1], device=cuda_device)}]
            ref = model(f[None], copy.copy(tgt), None)[0]
            got = graphed(f[None], copy.copy(tgt), None)[0]
            for key in ("pred_logits", "pred_boxes", "hs_embed"):
                scale = float(ref[key].abs().max())
                torch.testing.assert_close(got[key], ref[key], rtol=1e-4, atol=1e-5 * scale, msg=f"frame {i} {key}")
            prev = {k_: v.clone() for k_, v in ref.items() if torch.is_tensor(v)}
    assert graphed.captures == 3 and graphed.replays == 5               # track buckets 0, 8, 16


def test_graphed_train_step_equals_eager_for_vanilla_detection(cuda_device, strict_fp32):
    from trackformer_b200.train_step import TrainStep
    torch.manual_seed(0)
    model, criterion = df.build(False, False, device=str(cuda_device), enc_layers=2, dec_layers=3, dropout=0.0)
    model, criterion = model.to(cuda_device).train(), criterion.to(cuda_device).train()
    model_e = copy.deepcopy(model)
    g = torch.Generator().manual_seed(3)
    frames = [torch.randn(1, 3, 192, 256, generator=g).to(cuda_device) for _ in range(3)]
    graphed = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames[0])
    eager = TrainStep(model_e, criterion, None, use_graphs=False)
    for i, f in enumerate(frames):
        n = 4 + i
        gb = torch.Generator().manual_seed(10 + i)
        boxes = torch.cat([torch.rand(n, 2, generator=gb) * 0.5 + 0.25, torch.rand(n, 2, generator=gb) * 0.2 + 0.05], 1)
        tg = [{"boxes": boxes.to(cuda_device), "labels": torch.randint(0, 91, (n,), generator=gb).to(cuda_device)}]
        loss_g = graphed(f, tg)
        loss_e = eager(f, tg)
        torch.testing.assert_close(loss_g, loss_e, rtol=1e-4, atol=1e-4)
        scale = float(eager.flat_grad.abs().max())
        torch.testing.assert_close(graphed.flat_grad, eager.flat_grad, rtol=1e-3, atol=2e-4 * scale)
