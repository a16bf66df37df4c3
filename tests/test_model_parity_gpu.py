"""GPU model-level parity: the trackformer_b200 model on the real sm_90a kernels against golden outputs
recorded from the reference classes on CPU (tests/golden/make_golden_model.py).

Tolerance (BASELINE.json north_star): boxes / logits within 1e-3 relative of the reference; index
bookkeeping bit-exact.  Strict-fp32 runs (TF32 off) are held to that bar elementwise
(rtol 1e-3, atol 1e-3 x tensor scale); the TF32 run -- the arithmetic the benchmark uses for the dense
GEMMs/convolutions -- is held to the same bar on the final boxes and logits.
"""
import numpy as np
import pytest
import torch

import model_fixtures as mf
from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


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


def builder(dev):
    def build(tracking, multi_frame, **overrides):
        from trackformer_b200.model_factory import build_model, default_args
        torch.manual_seed(0)
        model, criterion, _ = build_model(default_args(tracking, multi_frame, device=str(dev), **overrides))
        return model, criterion
    return build


def check(res, gold, keys, rtol=1e-3, rel_atol=1e-3):
    worst = {}
    for k in keys:
        g = np.asarray(gold[k])
        scale = float(np.abs(g).max()) or 1.0
        np.testing.assert_allclose(np.asarray(res[k]), g, rtol=rtol, atol=rel_atol * scale, err_msg=k)
        worst[k] = float(np.abs(np.asarray(res[k]) - g).max() / scale)
    return worst


def test_detection_mini(dev, strict_fp32):
    gold = load_golden("det_mini", "model_")
    res = mf.run_detection(builder(dev), [(160, 224)], device=dev)
    assert res["image_digest"] == str(gold["image_digest"])
    print(check(res, gold, ["pred_logits", "pred_boxes", "hs_last_mean", "aux4_boxes", "memory0_mean"]))


def test_detection_c1_480x640(dev, strict_fp32):
    """BASELINE config[0]: single 3x480x640 frame, 4 levels, 300 queries."""
    gold = load_golden("det_c1_480x640", "model_")
    res = mf.run_detection(builder(dev), [(480, 640)], device=dev)
    assert res["image_digest"] == str(gold["image_digest"])
    print(check(res, gold, ["pred_logits", "pred_boxes", "hs_last_mean", "aux4_boxes"]))


def test_detection_c1_tf32(dev, tf32):
    gold = load_golden("det_c1_480x640", "model_")
    res = mf.run_detection(builder(dev), [(480, 640)], device=dev)
    print("tf32:", check(res, gold, ["pred_logits", "pred_boxes"], rtol=1e-3, rel_atol=1e-3))


def test_padded_batch(dev, strict_fp32):
    gold = load_golden("det_padded_batch", "model_")
    res = mf.run_detection(builder(dev), [(160, 224), (128, 192)], device=dev)
    print(check(res, gold, ["pred_logits", "pred_boxes", "hs_last_mean", "aux4_boxes", "memory0_mean"]))


def test_two_frame_tracking(dev, strict_fp32):
    gold = load_golden("track_two_frames", "model_")
    res = mf.run_two_frame_tracking(builder(dev), (160, 224), 12, device=dev)
    print(check(res, gold, ["f1_logits", "f1_boxes", "f2_logits", "f2_boxes", "f2_hs_mean"]))


def test_multi_frame_tracking_d36_l8(dev, strict_fp32):
    gold = load_golden("track_multi_frame", "model_")
    res = mf.run_two_frame_tracking(builder(dev), (128, 160), 9, device=dev, multi_frame=True)
    assert int(res["n_levels_memory"]) == 8
    print(check(res, gold, ["f1_logits", "f1_boxes", "f2_logits", "f2_boxes", "f2_hs_mean"]))


def test_train_step_losses_and_grads(dev, strict_fp32):
    gold = load_golden("train_step_det", "model_")
    res = mf.run_train_step(builder(dev), [(160, 224), (160, 224)], 6, device=dev)
    check(res, gold, [k for k in gold if k.startswith("loss/") and "class_error" not in k and "cardinality" not in k]
          + ["loss_total", "pred_logits", "pred_boxes"])
    for k in [k for k in gold if k.startswith("grad/")]:
        scale = float(np.abs(gold[k]).max())
        np.testing.assert_allclose(res[k], gold[k], rtol=5e-3, atol=2e-3 * max(scale, 1e-3), err_msg=k)
    np.testing.assert_allclose(res["grad_global_norm"], gold["grad_global_norm"], rtol=2e-3)


def test_tracking_train_step_bookkeeping_bit_exact(dev, strict_fp32):
    gold = load_golden("train_step_tracking", "model_")
    res = mf.run_train_step(builder(dev), [(128, 160)], 7, device=dev, tracking=True)
    for k in [k for k in gold if k.startswith("idx/")]:
        assert np.array_equal(res[k], gold[k]), k
    check(res, gold, ["loss_total", "loss/loss_ce", "loss/loss_bbox", "loss/loss_giou"])


# ---------------------------------------------------------------------------------------------------------
# BASELINE.json configs[1], [2], [4] at their FULL sizes: the configurations bench.py / tools/track_bench.py time.
# Strict fp32 is held to the elementwise 1e-3 bar; TF32 (the arithmetic the benchmark uses for the dense parts) to
# the same bar on the final boxes / logits, and its measured worst relative error is printed.
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_detection_c2_800x1333(dev, mode, request):
    request.getfixturevalue("strict_fp32" if mode == "fp32" else "tf32")
    gold = load_golden("det_c2_800x1333", "model_")
    res = mf.run_detection(builder(dev), [(800, 1333)], device=dev)
    assert res["image_digest"] == str(gold["image_digest"])
    keys = ["pred_logits", "pred_boxes"] + (["hs_last_mean", "aux4_boxes", "memory0_mean"] if mode == "fp32" else [])
    print(mode, check(res, gold, keys))


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_tracking_c3_two_frames_800x1333(dev, mode, request):
    """configs[2]: two frames 800x1333, 100 track + 300 object queries."""
    request.getfixturevalue("strict_fp32" if mode == "fp32" else "tf32")
    gold = load_golden("track_c3_800x1333", "model_")
    res = mf.run_two_frame_tracking(builder(dev), (800, 1333), 100, device=dev)
    keys = ["f1_logits", "f1_boxes", "f2_logits", "f2_boxes"] + (["f2_hs_mean"] if mode == "fp32" else [])
    print(mode, check(res, gold, keys))


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_tracking_c5_multi_frame_1080x1920(dev, mode, request):
    """configs[4] geometry: 1080x1920, multi-frame attention (hidden 288, D = 36, 8 decoder levels), 300 track + 500
    object queries."""
    request.getfixturevalue("strict_fp32" if mode == "fp32" else "tf32")
    gold = load_golden("track_c5_1080x1920", "model_")
    res = mf.run_two_frame_tracking(builder(dev), (1080, 1920), 300, device=dev, multi_frame=True)
    assert int(res["n_levels_memory"]) == 8
    keys = ["f1_logits", "f1_boxes", "f2_logits", "f2_boxes"] + (["f2_hs_mean"] if mode == "fp32" else [])
    print(mode, check(res, gold, keys))


def _grad_report(res, gold):
    rep = {}
    for k in [k for k in gold if k.startswith("grad/")]:
        a, b = np.asarray(res[k], np.float64).ravel(), np.asarray(gold[k], np.float64).ravel()
        rep[k[5:]] = (float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)),
                      float(a @ b / max(np.linalg.norm(a) * np.linalg.norm(b), 1e-30)))
    return rep


def test_train_step_c2_fp32(dev, strict_fp32):
    """configs[1] train step (forward + SetCriterion + backward, dropout 0) at 800x1333 against the reference."""
    gold = load_golden("train_step_c2", "model_")
    res = mf.run_train_step(builder(dev), [(800, 1333)], 20, device=dev)
    check(res, gold, [k for k in gold if k.startswith("loss/") and "class_error" not in k and "cardinality" not in k]
          + ["loss_total", "pred_logits", "pred_boxes"])
    for k in [k for k in gold if k.startswith("grad/")]:
        scale = float(np.abs(gold[k]).max())
        np.testing.assert_allclose(res[k], gold[k], rtol=5e-3, atol=2e-3 * max(scale, 1e-3), err_msg=k)
    np.testing.assert_allclose(res["grad_global_norm"], gold["grad_global_norm"], rtol=2e-3)
    print(_grad_report(res, gold))


def test_train_step_c2_tf32(dev, tf32):
    """The same step under TF32 dense math: outputs and losses to the 1e-3 bar, gradients by direction and size
    (a TF32 product carries ~5e-4 relative error per contraction, so elementwise gradient equality is not the bar)."""
    gold = load_golden("train_step_c2", "model_")
    res = mf.run_train_step(builder(dev), [(800, 1333)], 20, device=dev)
    print("tf32 outputs:", check(res, gold, ["pred_logits", "pred_boxes"]))
    for k in ["loss_total"] + [k for k in gold if k.startswith("loss/") and "class_error" not in k
                               and "cardinality" not in k]:
        np.testing.assert_allclose(res[k], gold[k], rtol=5e-3, atol=1e-4, err_msg=k)
    np.testing.assert_allclose(res["grad_global_norm"], gold["grad_global_norm"], rtol=2e-2)
    rep = _grad_report(res, gold)
    print("tf32 gradients (max rel err, cosine):", rep)
    for k, (err, cos) in rep.items():
        # sampling-offset gradients are sums of DIFFERENCES of neighbouring value rows (the bilinear derivative), so a
        # TF32 value projection (~5e-4 relative per element) shows up amplified there, hence
        # the looser cosine bound for those tensors
        assert cos > (0.995 if "sampling_offsets" in k else 0.999), (k, err, cos)


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_bench_pipeline_one_step_c2(dev, mode, request):
    """ONE step of the exact bench.py pipeline -- full-step CUDA graph (forward + device Hungarian matching + loss +
    backward + gradient gather), flat one-pass clip + AdamW kernel with the reference's three lr groups -- at 800x1333
    (dropout 0) against the reference's loss and its UPDATED weights (engine.py:147-151 + train.py:100-119)."""
    request.getfixturevalue("strict_fp32" if mode == "fp32" else "tf32")
    from trackformer_b200.flat_adamw import reference_param_groups
    from trackformer_b200.train_step import TrainStep
    gold = load_golden("train_step_c2", "model_")
    model, criterion = builder(dev)(False, False, dropout=0.0)
    mf.canonical_weights_(model, 0)
    model.to(dev).train()
    criterion.to(dev).train()
    frames = mf.make_images(3, [(800, 1333)], dev)[0][None]
    targets = mf.make_targets(4, 1, 20, 1, dev)
    named = dict(model.named_parameters())
    before = {k: named[k].detach().clone() for k in mf.GRAD_KEYS if k in named}
    for k, b in before.items():
        np.testing.assert_array_equal(b.cpu().numpy(), gold["param_before/" + k], err_msg=k)
    step = TrainStep(model, criterion, None, max_norm=0.1, use_graphs=True, example_frames=frames,
                     example_targets=targets, flat_adamw={"groups": reference_param_groups(model)})
    assert step.g_full is not None
    # capture warm-ups ran backward passes but no optimizer step: weights are still the canonical ones
    loss = float(step(frames, targets))
    np.testing.assert_allclose(loss, float(gold["loss_total"]), rtol=1e-3 if mode == "fp32" else 5e-3)
    lr = {k: (2e-5 if "sampling_offsets" in k or "reference_points" in k else 2e-4) for k in before}
    worst = {}
    for k, b in before.items():
        ours = (named[k].detach() - b).cpu().numpy().ravel()
        ref = (gold["param/" + k] - gold["param_before/" + k]).ravel()
        # first AdamW step: |update| ~ lr per element wherever |g| >> eps, so compare in units of lr; elements whose
        # gradient is numerically zero may legitimately differ in sign
        ok = np.abs(ours - ref) <= 0.05 * lr[k]
        worst[k] = float(ok.mean())
        if mode == "fp32":
            assert ok.mean() >= 0.98, (k, ok.mean())
        else:
            # the first AdamW update is lr * sign(g) wherever |g| >> eps, so an element whose gradient is below the TF32
            # rounding noise of the step (~5e-4 relative per contraction, measured against the largest gradient of the
            # tensor) may flip by a whole lr: hold the elements that carry signal to the bar, report the rest
            gref = np.abs(gold["grad/" + k]).ravel()
            sig = gref >= 3e-3 * gref.max()
            assert ok[sig].mean() >= (0.93 if "sampling_offsets" in k else 0.97), (k, float(ok[sig].mean()), float(sig.mean()))
            assert ok.mean() >= 0.85, (k, ok.mean())
    print(mode, "fraction of updated elements within 5% of lr:", worst)
