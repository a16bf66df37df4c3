"""CPU tests of ``TrainStep(..., masks=True)``: the segmentation models trained with the mask head run on the last
layer's matched rows only, against the reference composition (``model(samples, targets)`` with the all-row head, then
``SetCriterion``, then backward) and the recorded training-step fixtures; the ragged ``mask_logits`` form; the criterion's
exposed matching; and argument validation of the ragged mask-head entry points.

The MSDeformAttn core has no CPU path: the oracle's torch restatement stands in for it, as in test_track_train_cpu.py."""
import copy
import ctypes

import numpy as np
import pytest
import torch

import detr_fixtures as df
import model_fixtures as mf
import segm_fixtures as sf
from conftest import load_golden
from test_model_parity_cpu import build, oracle_op  # noqa: F401  (fixture)
from test_track_train_cpu import assert_same_bookkeeping, flat_of, tracking_batch

SMALL = dict(enc_layers=1, dec_layers=2, num_queries=20, dropout=0.0)
VANILLA_SMALL = dict(enc_layers=1, dec_layers=2, num_queries=12, dropout=0.0)


def build_segm(kind, tracking, **overrides):
    if kind == "deformable":
        return build(tracking, False, masks=True, **dict(SMALL, **overrides))
    return df.build(tracking, False, masks=True, **dict(VANILLA_SMALL, **overrides))


def add_masks(targets, size, seed):
    g = torch.Generator().manual_seed(seed)
    h, w = size
    for t in targets:
        for tt in (t, t.get("prev_target")):
            if tt is not None:
                tt["masks"] = torch.rand(len(tt["boxes"]), h, w, generator=g) > 0.5
    return targets


def reference_step(model, criterion, frames, targets):
    out, targets_out, _, _, _ = model(frames, targets)
    loss_dict = criterion(out, targets_out)
    wd = criterion.weight_dict
    total = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
    model.zero_grad(set_to_none=True)
    total.backward()
    return total.detach(), targets_out


def make_step(model, criterion, bucket=1):
    from trackformer_b200.train_step import TrainStep
    return TrainStep(model, criterion, None, use_graphs=False, track_bucket=bucket, masks=True)


def assert_step_matches(step, loss, ref, ref_loss):
    torch.testing.assert_close(loss, ref_loss, rtol=1e-5, atol=1e-6)
    ref_flat = flat_of(step, ref)
    torch.testing.assert_close(step.flat_grad, ref_flat, rtol=2e-4, atol=1e-6 * float(ref_flat.abs().max()))
    head = torch.zeros_like(step.flat_grad, dtype=torch.bool)
    for v in step._mask_views:
        o = (v.data_ptr() - step.flat_grad.data_ptr()) // 4
        head[o:o + v.numel()] = True
    assert float(step.flat_grad[head].abs().max()) > 0                  # the mask head trained
    return head


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["deformable", "vanilla"])
def test_ragged_mask_logits_equal_the_all_row_head(oracle_op, kind):
    model, _ = build_segm(kind, False)
    mf.canonical_weights_(model, 0)
    model.eval()
    frames = mf.make_images(1, [(96, 128), (80, 112), (96, 96)])
    with torch.no_grad():
        out, _, features, memory, hs = model.detect(frames)
        full = model.mask_logits(features, memory, hs)
        src = torch.tensor([3, 0, 7, 5, 2, 9])
        sizes = [4, 0, 2]                                              # the middle image owns no row
        got = model.mask_logits(features, memory, hs, rows=(src, sizes))
    bat = torch.tensor([0, 0, 0, 0, 2, 2])
    assert got.shape == (6, *full.shape[-2:])
    torch.testing.assert_close(got, full[bat, src], rtol=1e-5, atol=1e-6)
    with torch.no_grad():
        none = model.mask_logits(features, memory, hs, rows=(src[:0], [0, 0, 0]))
    assert none.shape == (0, *full.shape[-2:])


@pytest.mark.parametrize("kind", ["deformable", "vanilla"])
@pytest.mark.parametrize("zero_boxes", [False, True], ids=["boxes", "zero_box_image"])
def test_detection_step_equals_the_reference_composition(oracle_op, kind, zero_boxes):
    model, criterion = build_segm(kind, False)
    mf.canonical_weights_(model, 1)
    model.train()
    ref = copy.deepcopy(model)
    size = (96, 128)
    frames = torch.stack(mf.make_images(4, [size, size]))
    targets = add_masks(mf.make_targets(5, 2, 5, 1), size, 6)
    if zero_boxes:                      # the criterion's per-layer fallback: the mask branch takes its indices
        targets[1] = {k: v[:0] if k in ("boxes", "labels", "track_ids", "masks") else v for k, v in targets[1].items()}
    step = make_step(model, criterion)
    assert step._tracking_route(targets) == "detect"
    loss = step(frames, targets)
    ref_loss, _ = reference_step(ref, criterion, frames, copy.deepcopy(targets))
    assert_step_matches(step, loss, ref, ref_loss)


@pytest.mark.parametrize("kind", ["deformable", "vanilla"])
@pytest.mark.parametrize("bucket", [1, 8])
def test_tracking_step_equals_the_reference_composition(oracle_op, kind, bucket):
    model, criterion = build_segm(kind, True)
    mf.canonical_weights_(model, 2)
    model.train()
    ref = copy.deepcopy(model)
    frames, targets = tracking_batch(2, sizes=((96, 128), (96, 128)))
    targets = add_masks(targets, (96, 128), 7)
    ref_targets = copy.deepcopy(targets)
    step = make_step(model, criterion, bucket)
    assert step._tracking_route(targets) == "track"
    torch.manual_seed(11)
    loss = step(frames, targets)
    torch.manual_seed(11)
    ref_loss, ref_targets = reference_step(ref, criterion, frames, ref_targets)
    assert_same_bookkeeping(targets, ref_targets)
    k = len(targets[0]["track_query_boxes"])
    assert k > 0 and (bucket == 1 or k % bucket != 0)                 # track queries, and fillers when bucketed
    assert_step_matches(step, loss, ref, ref_loss)


def test_freeze_detr_trains_only_the_mask_head(oracle_op):
    model, criterion = build_segm("deformable", True, freeze_detr=True)
    mf.canonical_weights_(model, 3)
    model.train()
    ref = copy.deepcopy(model)
    frames, targets = tracking_batch(3)
    targets = add_masks(targets, (96, 128), 8)
    ref_targets = copy.deepcopy(targets)
    step = make_step(model, criterion, 4)
    names = {id(p): n for n, p in model.named_parameters()}
    assert {names[id(p)].split(".")[0] for p in step.params} == {"mask_head", "bbox_attention"}
    torch.manual_seed(4)
    loss = step(frames, targets)
    torch.manual_seed(4)
    ref_loss, _ = reference_step(ref, criterion, frames, ref_targets)
    head = assert_step_matches(step, loss, ref, ref_loss)
    assert float(step.flat_grad[~head].abs().sum()) == 0.0


@pytest.mark.parametrize("case", ["model_segm_det_mini", "detr_segm_det_mini"])
def test_recorded_training_gradients_through_train_step(oracle_op, case):
    """tests/golden/{model,detr}_segm_det_mini.npz: the reference's own training step of DeformableDETRSegm / DETRSegm
    on a padded two-image batch, reproduced by TrainStep(masks=True)."""
    from trackformer_b200.train_step import TrainStep
    gold = load_golden(case.split("_", 1)[1], case.split("_", 1)[0] + "_")
    if case.startswith("model"):
        model, criterion = build(False, False, dropout=0.0, masks=True)
    else:
        model, criterion = df.build(False, False, dropout=0.0, masks=True)
    mf.canonical_weights_(model, 0)
    model.train()
    imgs = mf.make_images(3, sf.SIZES)
    targets = sf.mask_targets(4, sf.SIZES, sf.N_BOXES)
    step = TrainStep(model, criterion, None, use_graphs=False, masks=True)
    loss = step(imgs, targets)
    np.testing.assert_allclose(float(loss), gold["loss_total"], rtol=1e-3, atol=2e-5)
    named = dict(model.named_parameters())
    for k in sf.GRAD_KEYS:
        np.testing.assert_allclose(named[k].grad.numpy(), gold["grad/" + k], rtol=1e-3, atol=2e-5, err_msg=k)
    head = sum(float((p.grad.double() ** 2).sum()) for n, p in named.items()
               if n.startswith(("mask_head.", "bbox_attention.")))
    np.testing.assert_allclose(np.sqrt(head), gold["grad_mask_head_norm"], rtol=1e-3)
    np.testing.assert_allclose(float(step.flat_grad.double().norm()), gold["grad_global_norm"], rtol=1e-3)


def test_forced_matching_with_masks_equals_forward_and_exposes_the_last_layer():
    from test_track_train_cpu import random_tracking_targets
    _, criterion = build_segm("deformable", True)
    g = torch.Generator().manual_seed(5)
    nq, n_track, n_layers = 20, 4, 2
    targets = [random_tracking_targets(g, 6, n_track, 1, nq), random_tracking_targets(g, 5, n_track, 0, nq)]
    for t in targets:
        t["masks"] = torch.rand(len(t["boxes"]), 40, 56, generator=g) > 0.5
    logits = torch.randn(n_layers, 2, n_track + nq, 20, generator=g)
    boxes = torch.rand(n_layers, 2, n_track + nq, 4, generator=g)
    pred_masks = torch.randn(2, n_track + nq, 10, 14, generator=g)
    ref = criterion(dict(pred_logits=logits[-1], pred_boxes=boxes[-1], pred_masks=pred_masks,
                         aux_outputs=[{"pred_logits": logits[0], "pred_boxes": boxes[0]}]), targets)
    got = criterion.forward_stacked(logits, boxes, targets, pred_masks=pred_masks, track_queries=True)
    assert got.stacked is not None and set(got) == set(ref)            # the stacked (forced) route
    for k in ref:
        torch.testing.assert_close(got[k], ref[k], rtol=1e-5, atol=1e-6, msg=k)
    bat, src, tgt = got.matched
    assert got.matched_sizes == [6, 5]
    indices = criterion.matcher({"pred_logits": logits[-1], "pred_boxes": boxes[-1]}, targets)
    assert torch.equal(bat, torch.tensor([0] * 6 + [1] * 5))
    assert torch.equal(src, torch.cat([s for s, _ in indices]))
    assert torch.equal(tgt, torch.cat([indices[0][1], indices[1][1] + 6]))
    # without pred_masks the mask terms are left to the caller; everything else is unchanged
    rest = criterion.forward_stacked(logits, boxes, targets, track_queries=True)
    assert set(rest) == set(ref) - {"loss_mask", "loss_dice"}
    for k in rest:
        torch.testing.assert_close(rest[k], got[k], rtol=0, atol=0, msg=k)


def test_mask_models_still_need_the_keyword():
    from trackformer_b200.train_step import TrainStep
    model, criterion = build_segm("deformable", False)
    with pytest.raises(NotImplementedError, match="masks=True"):
        TrainStep(model, criterion, use_graphs=False)
    plain, plain_criterion = build(False, False, **SMALL)
    with pytest.raises(ValueError, match="segmentation model"):
        TrainStep(plain, plain_criterion, use_graphs=False, masks=True)


def test_ragged_entry_points_validate_arguments():
    from trackformer_b200 import _build as b
    lib = ctypes.CDLL(b.build_library())
    vp, i, i64, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, vp)
    odd = ctypes.c_void_p(ctypes.addressof(buf) + 4)
    attn = lib.tfb200_mask_attn_rows_fwd_f32
    attn.argtypes = [vp] * 5 + [i, i, i, i, f, vp]
    assert attn(p, p, None, None, p, 1, 1, 4, 8, 1.0, None) == -1          # no row_offsets
    assert attn(None, p, None, p, p, 1, 1, 4, 8, 1.0, None) == -1          # rows but no q
    assert attn(p, p, None, p, p, -1, 0, 4, 8, 1.0, None) == -2            # B < 0
    assert attn(p, p, None, p, p, 0, 3, 4, 8, 1.0, None) == -2             # rows without images
    assert attn(p, p, None, p, p, 1, 1, 0, 8, 1.0, None) == -2             # HW = 0
    assert attn(p, p, None, p, p, 1, 1, 4, 257, 1.0, None) == -2           # beyond the shared-memory stage
    assert attn(odd, p, None, p, p, 1, 1, 4, 8, 1.0, None) == -2           # q not 16-byte aligned
    assert attn(None, p, None, p, None, 2, 0, 4, 8, 1.0, None) == 0        # P = 0: a no-op
    attn_bwd = lib.tfb200_mask_attn_rows_bwd_f32
    attn_bwd.argtypes = [vp] * 8 + [i, i, i, i, f, vp]
    assert attn_bwd(p, p, p, p, p, p, p, None, 1, 1, 4, 8, 1.0, None) == -1  # no dk
    assert attn_bwd(p, p, p, p, p, p, p, odd, 1, 1, 4, 8, 1.0, None) == -2   # dk not 16-byte aligned
    assert attn_bwd(p, p, p, p, p, p, p, p, 0, 1, 4, 8, 1.0, None) == -2     # rows without images
    assert attn_bwd(p, p, p, p, p, p, p, p, 0, 0, 4, 8, 1.0, None) == 0      # nothing at all
    gn = lib.tfb200_group_norm_relu_rows_fwd_f32
    gn.argtypes = [vp] * 8 + [i, i, i64, i, i, f, vp]
    assert gn(p, None, p, p, p, p, p, p, 2, 2, 16, 16, 8, 1e-5, None) == -1      # no addend
    assert gn(p, p, None, p, p, p, p, p, 2, 2, 16, 16, 8, 1e-5, None) == -1      # no row_offsets
    assert gn(p, p, p, p, p, p, p, p, 2, 2, 16, 18, 8, 1e-5, None) == -2         # C % groups
    assert gn(p, p, p, p, p, p, p, p, 2, 2, 16, 8 * 264, 8, 1e-5, None) == -2    # > 256 channels per group
    assert gn(p, p, p, p, p, p, p, p, 2, -1, 16, 16, 8, 1e-5, None) == -2        # P < 0
    gn_bwd = lib.tfb200_group_norm_relu_rows_bwd_f32
    gn_bwd.argtypes = [vp] * 12 + [i, i, i64, i, i, vp]
    assert gn_bwd(*([p] * 9), None, p, p, 2, 2, 16, 16, 8, None) == -1          # no daddend
    assert gn_bwd(*([p] * 12), 0, 2, 16, 16, 8, None) == -2                     # rows without images
    up = lib.tfb200_upsample_add_rows_fwd_f32
    up.argtypes = [vp] * 4 + [i] * 7 + [vp]
    assert up(p, None, p, p, 2, 3, 4, 4, 8, 8, 16, None) == -1                  # no per-image operand
    assert up(p, p, p, p, 2, 3, 0, 4, 8, 8, 16, None) == -2                     # Hi = 0
    up_bwd = lib.tfb200_upsample_add_rows_bwd_f32
    up_bwd.argtypes = [vp] * 4 + [i] * 7 + [vp]
    assert up_bwd(p, None, p, p, 2, 3, 4, 4, 8, 8, 16, None) == -1              # no row_offsets
    assert up_bwd(p, p, p, p, -2, 0, 4, 4, 8, 8, 16, None) == -2                # B < 0


def test_ragged_bindings_reject_cpu_tensors():
    from trackformer_b200 import ext
    m = ext.load()
    off = torch.tensor([0, 2], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.mask_attn_rows_forward(torch.zeros(2, 256), torch.zeros(1, 4, 256), None, off, 8, 1.0)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.group_norm_relu_rows_forward(torch.zeros(2, 16, 4, 4), torch.zeros(1, 16, 4, 4), off, torch.ones(16),
                                       torch.zeros(16), 8, 1e-5)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.upsample_add_rows_forward(torch.zeros(2, 16, 4, 4), torch.zeros(1, 16, 8, 8), off)
