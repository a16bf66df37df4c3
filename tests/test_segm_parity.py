"""Parity of the segmentation models with the reference: trackformer_b200 against fixtures recorded from the
reference classes on CPU (tests/golden/make_golden_segm.py, model_segm_*.npz).

CPU cases run the product's CPU path (the MSDeformAttn core replaced by the oracle's torch restatement, as in
tests/test_model_parity_cpu.py) at that file's tolerances; GPU cases run the sm_90a kernels at the tolerances of
tests/test_model_parity_gpu.py, strict fp32 and TF32.
"""
import numpy as np
import pytest
import torch

import segm_fixtures as sf
from conftest import load_golden


@pytest.fixture()
def oracle_op(monkeypatch):
    from oracle.torch_ref import msda_core_torch
    import trackformer_b200.msda_module as mm

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    monkeypatch.setattr(mm, "MSDeformAttnFunction", _OracleFn)


def builder(device):
    def build(tracking, multi_frame, **overrides):
        from trackformer_b200.model_factory import build_model, default_args
        torch.manual_seed(0)
        model, criterion, _ = build_model(default_args(tracking, multi_frame, device=str(device), **overrides))
        return model, criterion
    return build


def _post():
    from trackformer_b200.segmentation import PostProcessSegm
    return PostProcessSegm


def check_abs(res, gold, keys, rtol=1e-3, atol=2e-5):
    for k in keys:
        np.testing.assert_allclose(np.asarray(res[k]), gold[k], rtol=rtol, atol=atol, err_msg=k)


def check_scaled(res, gold, keys, rtol=1e-3, rel_atol=1e-3):
    for k in keys:
        g = np.asarray(gold[k])
        scale = float(np.abs(g).max()) or 1.0
        np.testing.assert_allclose(np.asarray(res[k]), g, rtol=rtol, atol=rel_atol * scale, err_msg=k)


OUT_KEYS = ["pred_masks_rows", "pred_masks_mean", "loss_total", "loss_mask", "loss_dice"]
GRAD_KEYS = ["grad/" + k for k in sf.GRAD_KEYS] + ["grad_mask_head_norm", "grad_global_norm"]


def _segm_outputs_agree(res, gold, strict):
    """Binary masks may flip only where the reference probability sits at the threshold."""
    for i in range(len(sf.SIZES)):
        got, ref = res[f"segm/{i}"], gold[f"segm/{i}"]
        assert got.shape == ref.shape and got.dtype == ref.dtype
        near = np.abs(gold[f"segm_probs/{i}"] - 0.5) < (1e-5 if strict else 1e-3)
        assert np.array_equal(got[~near], ref[~near])
        np.testing.assert_allclose(res[f"segm_probs/{i}"], gold[f"segm_probs/{i}"], rtol=1e-4, atol=1e-5)


def test_state_dict_keys_equal_reference():
    gold = load_golden("segm_det_mini", "model_")
    model, _ = builder("cpu")(False, False, masks=True)
    assert sorted(model.state_dict()) == list(gold["state_dict_keys"])
    gold = load_golden("segm_track_two_frames", "model_")
    model, _ = builder("cpu")(True, False, masks=True)
    assert sorted(model.state_dict()) == list(gold["state_dict_keys"])


def test_segm_train_step_cpu(oracle_op):
    gold = load_golden("segm_det_mini", "model_")
    res = sf.run_segm_train_step(builder("cpu"), _post())
    check_abs(res, gold, OUT_KEYS + GRAD_KEYS)
    _segm_outputs_agree(res, gold, strict=True)


def test_segm_two_frames_cpu(oracle_op):
    gold = load_golden("segm_track_two_frames", "model_")
    res = sf.run_segm_two_frames(builder("cpu"))
    check_abs(res, gold, ["f1_masks_rows", "f1_masks_mean", "f2_masks_rows", "f2_masks_mean", "f2_boxes"])


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def tf32_mode(request):
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = request.param
    yield request.param
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.mark.gpu
@pytest.mark.parametrize("tf32_mode", [False, True], ids=["strict_fp32", "tf32"], indirect=True)
def test_segm_train_step_gpu(cuda_device, tf32_mode):
    gold = load_golden("segm_det_mini", "model_")
    res = sf.run_segm_train_step(builder(cuda_device), _post(), device=cuda_device)
    if tf32_mode:
        check_scaled(res, gold, ["pred_masks_mean", "loss_mask", "loss_dice"], rtol=1e-2, rel_atol=1e-2)
        return
    check_scaled(res, gold, OUT_KEYS)
    for k in ["grad/" + k for k in sf.GRAD_KEYS]:               # the gradient rule of test_model_parity_gpu.py
        scale = float(np.abs(gold[k]).max())
        np.testing.assert_allclose(res[k], gold[k], rtol=5e-3, atol=2e-3 * max(scale, 1e-3), err_msg=k)
    for k in ("grad_mask_head_norm", "grad_global_norm"):
        np.testing.assert_allclose(res[k], gold[k], rtol=2e-3, err_msg=k)
    _segm_outputs_agree(res, gold, strict=False)


@pytest.mark.gpu
@pytest.mark.parametrize("tf32_mode", [False, True], ids=["strict_fp32", "tf32"], indirect=True)
def test_segm_two_frames_gpu(cuda_device, tf32_mode):
    gold = load_golden("segm_track_two_frames", "model_")
    res = sf.run_segm_two_frames(builder(cuda_device), device=cuda_device)
    keys = ["f1_masks_mean", "f2_masks_mean", "f2_boxes"]
    if tf32_mode:
        check_scaled(res, gold, keys, rtol=1e-2, rel_atol=1e-2)
    else:
        check_scaled(res, gold, keys + ["f1_masks_rows", "f2_masks_rows"])
