"""Two-stage Deformable DETR on the CPU: construction, refusals, the host build of the proposal / selection routines
(tests/host_build/two_stage_host.cpp, the code of csrc/two_stage.cu) and the product model against fixtures recorded from
the reference (tests/golden/make_golden_two_stage.py).

As in test_model_parity_cpu.py, only the MSDeformAttn core is replaced by the oracle's torch restatement; the two-stage
branch runs its CPU route (the reference's torch ops).
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
import host_twin
import two_stage_fixtures as tf

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


@pytest.fixture()
def oracle_op(monkeypatch):
    from oracle.torch_ref import msda_core_torch
    import trackformer_b200.msda_module as mm

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    monkeypatch.setattr(mm, "MSDeformAttnFunction", _OracleFn)


def build(tracking, multi_frame, **overrides):
    from trackformer_b200.model_factory import build_model, default_args
    torch.manual_seed(0)
    model, criterion, _ = build_model(default_args(tracking, multi_frame, device="cpu", **overrides))
    return model, criterion


def check(res, gold, keys, rtol=1e-3, atol=2e-5):
    for k in keys:
        np.testing.assert_allclose(np.asarray(res[k]), gold[k], rtol=rtol, atol=atol, err_msg=k)


# The sine embedding is held to an absolute bound: libm and torch's vectorised exp / sin / cos each round within 1 ulp,
# and a 1-ulp change of sigmoid(box) moves the argument (up to 2 pi) by up to 4.8e-7 -- many ulps of an output near 0.
EMBED_ATOL = 4 * float(np.spacing(np.float32(2 * np.pi)))


def ulps(a, b):
    """distance in units in the last place between fp32 arrays (equal infinities: 0)"""
    def key(x):
        i = np.ascontiguousarray(x, dtype=np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


# ---- construction -------------------------------------------------------------------------------------------------
def test_state_dict_keys_and_shapes_equal_the_reference():
    gold = load_golden("state_dict", "two_stage_")
    model, _ = build(False, False, two_stage=True)
    sd = model.state_dict()
    assert list(sd) == list(gold["keys"])
    assert [",".join(map(str, v.shape)) for v in sd.values()] == list(gold["shapes"])
    assert "transformer.reference_points.weight" not in sd and sd["query_embed.weight"].shape == (300, 256)
    assert "transformer.decoder.class_embed.6.bias" in sd and "transformer.decoder.bbox_embed.6.layers.2.bias" in sd
    g = torch.Generator().manual_seed(0)
    ref_layout = {k: torch.randn([int(d) for d in s.split(",") if d], generator=g) if s else torch.randn((), generator=g)
                  for k, s in zip(gold["keys"], gold["shapes"])}
    ref_layout = {k: v.to(sd[k].dtype) for k, v in ref_layout.items()}
    model.load_state_dict(ref_layout, strict=True)
    # the aliases share one tensor, as in the reference
    assert model.transformer.decoder.class_embed[6].weight is model.class_embed[6].weight


def test_box_heads_and_bias_init():
    model, criterion = build(False, False, two_stage=True)
    assert len(model.class_embed) == len(model.bbox_embed) == 7
    for box_embed in model.bbox_embed:
        assert torch.all(box_embed.layers[-1].bias[2:] == 0)
    for k in ("loss_ce", "loss_bbox", "loss_giou"):
        assert criterion.weight_dict[k + "_enc"] == criterion.weight_dict[k]


def test_two_stage_without_box_refinement_raises():
    with pytest.raises(ValueError, match="with_box_refine"):
        build(False, False, two_stage=True, with_box_refine=False)


@pytest.mark.parametrize("masks", [False, True])
def test_tracking_classes_refuse_two_stage(masks):
    with pytest.raises(NotImplementedError, match="track-query concatenation"):
        build(True, False, two_stage=True, masks=masks)


@pytest.mark.parametrize("separate", [True, False])
def test_multi_frame_attention_refuses_two_stage(separate):
    with pytest.raises(NotImplementedError, match="multi-frame"):
        build(False, True, two_stage=True, multi_frame_attention_separate_encoder=separate, hidden_dim=256)


def test_train_step_refuses_two_stage_segmentation():
    from trackformer_b200.train_step import TrainStep
    model, criterion = build(False, False, two_stage=True, masks=True)
    with pytest.raises(NotImplementedError, match="two-stage segmentation"):
        TrainStep(model, criterion, use_graphs=False, masks=True)


# ---- host build of the kernels' routines --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    lib = host_twin.build("two_stage_host", tmp_path_factory.mktemp("two_stage_host"))
    lib.tfb200_two_stage_proposals_host.restype = ctypes.c_int
    lib.tfb200_two_stage_select_host.restype = ctypes.c_int
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def host_proposals(lib, mask, hw, memory=None):
    b, s = mask.shape
    hw32 = np.ascontiguousarray(hw, dtype=np.int32).reshape(-1)
    prop = np.empty((b, s, 4), np.float32)
    valid = np.empty((b, s), np.uint8)
    c = 0 if memory is None else memory.shape[-1]
    masked = None if memory is None else np.empty_like(memory)
    rc = lib.tfb200_two_stage_proposals_host(_ptr(np.ascontiguousarray(mask, np.uint8)),
                                             None if memory is None else _ptr(memory),
                                             None if memory is None else _ptr(masked), _ptr(prop), _ptr(valid),
                                             b, s, len(hw32) // 2, c, _ptr(hw32))
    assert rc == 0
    return prop, valid, masked


def host_select(lib, logits, unact, k):
    from trackformer_b200.deformable_transformer import proposal_dim_t
    b, s, c = logits.shape
    dim_t = proposal_dim_t("cpu").numpy()
    keys = np.empty((b, s), np.uint32)
    index = np.empty((b, k), np.int64)
    boxes, ref = np.empty((b, k, 4), np.float32), np.empty((b, k, 4), np.float32)
    embed = np.empty((b, k, 512), np.float32)
    rc = lib.tfb200_two_stage_select_host(_ptr(np.ascontiguousarray(logits, np.float32)),
                                          _ptr(np.ascontiguousarray(unact, np.float32)), _ptr(dim_t), _ptr(keys),
                                          _ptr(index), _ptr(boxes), _ptr(ref), _ptr(embed), b, s, c, k)
    assert rc == 0
    return index, boxes, ref, embed


CASES = ["det_mini", "det_padded_batch", "det_800x1333", "train_step_det"]


@pytest.mark.parametrize("case", CASES)
def test_host_proposals_match_reference(host_lib, case):
    gold = load_golden(case, "two_stage_")
    prop, valid, _ = host_proposals(host_lib, gold["mask"], gold["hw"])
    ref_valid = np.isfinite(gold["prop"]).all(-1)
    assert np.array_equal(valid.astype(bool), ref_valid)
    assert np.array_equal(np.isinf(prop), np.isinf(gold["prop"]))
    assert ulps(prop, gold["prop"]).max() <= 2
    if case == "det_padded_batch":
        assert gold["mask"].any() and not ref_valid[gold["mask"].astype(bool)].any()


def test_host_masked_memory(host_lib):
    gold = load_golden("det_padded_batch", "two_stage_")
    mem = np.random.default_rng(0).standard_normal(gold["mask"].shape + (8,)).astype(np.float32)
    _, valid, masked = host_proposals(host_lib, gold["mask"], gold["hw"], mem)
    np.testing.assert_array_equal(masked, np.where(valid[..., None] == 1, mem, 0))


@pytest.mark.parametrize("case", CASES)
def test_host_selection_matches_reference(host_lib, case):
    gold = load_golden(case, "two_stage_")
    logit0, sel = gold["enc_logit0"], gold["selected"]
    b, s = logit0.shape
    k = sel.shape[1]
    unact = np.full((b, s, 4), np.nan, np.float32)
    for i in range(b):
        unact[i, sel[i]] = gold["topk_unact"][i]
    index, boxes, ref, embed = host_select(host_lib, logit0[..., None], unact, k)
    for i in range(b):
        # same values in the same order; tokens of exactly tied logits (invalid or padded) compare as sets
        np.testing.assert_array_equal(logit0[i, index[i]], logit0[i, sel[i]])
        for v in np.unique(logit0[i, sel[i]]):
            assert set(index[i][logit0[i, index[i]] == v]) <= set(np.flatnonzero(logit0[i] == v))
        tie = logit0[i, sel[i][-1]]
        if (logit0[i] == tie).sum() > 1:            # the lowest token indices of the boundary tie are taken
            need = int((logit0[i, index[i]] == tie).sum())
            assert sorted(index[i][logit0[i, index[i]] == tie]) == list(np.flatnonzero(logit0[i] == tie)[:need])
    np.testing.assert_array_equal(boxes, np.take_along_axis(unact, index[..., None], 1))
    assert ulps(ref, 1 / (1 + np.exp(-boxes.astype(np.float64)))).max() <= 2
    n = gold["embed_rows"].shape[1]
    assert np.abs(embed[:, :n] - gold["embed_rows"]).max() <= EMBED_ATOL


def test_host_selection_ties_take_the_lower_index(host_lib):
    rng = np.random.default_rng(3)
    logits = rng.standard_normal((2, 5000, 3)).astype(np.float32)
    logits[:, 100:4000:7, 0] = 2.5                    # 557 exact ties straddling k
    logits[1, 17, 0] = np.inf
    logits[1, 18, 0] = -0.0
    unact = rng.standard_normal((2, 5000, 4)).astype(np.float32)
    unact[:, 100:4000:7] = np.inf
    index, boxes, ref, embed = host_select(host_lib, logits, unact, 300)
    for b in range(2):
        order = np.lexsort((np.arange(5000), -logits[b, :, 0].astype(np.float64)))[:300]
        np.testing.assert_array_equal(index[b], order)
    assert np.isinf(boxes).any() and np.all(ref[np.isinf(boxes)] == 1.0) and np.isfinite(embed).all()


# ---- product model on the CPU ---------------------------------------------------------------------------------------
def _selected_equal(res, gold):
    np.testing.assert_array_equal(np.sort(res["selected"], 1), np.sort(gold["selected"], 1))


@pytest.mark.parametrize("case,sizes,seed", [("det_mini", [(160, 224)], 0),
                                             ("det_padded_batch", [(160, 224), (128, 192)], 1)])
def test_detection_matches_reference(oracle_op, case, sizes, seed):
    gold = load_golden(case, "two_stage_")
    res = tf.run_detection(build, sizes, seed=seed)
    assert res["image_digest"] == str(gold["image_digest"])
    _selected_equal(res, gold)
    np.testing.assert_array_equal(res["rows"], gold["rows"])
    check(res, gold, ["pred_logits", "pred_boxes", "aux0_boxes", "aux0_logits", "hs_last_mean", "enc_logits_rows",
                      "enc_boxes_rows", "enc_logit0"])


def test_segmentation_matches_reference(oracle_op):
    gold = load_golden("segm_det_mini", "two_stage_")
    res = tf.run_detection(build, [(160, 224)], masks=True)
    _selected_equal(res, gold)
    check(res, gold, ["pred_logits", "pred_boxes", "enc_logits_rows", "enc_boxes_rows", "pred_masks_mean"])


def test_train_step_losses_and_grads_match_reference(oracle_op):
    gold = load_golden("train_step_det", "two_stage_")
    res = tf.run_train_step(build, [(160, 224), (160, 224)], 6, seed=tf.TRAIN_STEP_SEED)
    _selected_equal(res, gold)
    losses = [k for k in gold if k.startswith("loss/")]
    assert {"loss/loss_ce_enc", "loss/loss_bbox_enc", "loss/loss_giou_enc", "loss/cardinality_error_enc"} <= set(losses)
    assert set(losses) == {k for k in res if k.startswith("loss/")}
    check(res, gold, losses + ["loss_total", "pred_logits", "pred_boxes"])
    for k in [k for k in gold if k.startswith("grad/")]:
        scale = float(np.abs(gold[k]).max())
        np.testing.assert_allclose(res[k], gold[k], rtol=2e-3, atol=2e-4 * max(scale, 1e-3), err_msg=k)
    for k in [k for k in gold if k.startswith("gradnorm/")]:
        np.testing.assert_allclose(res[k], gold[k], rtol=2e-3, err_msg=k)


def test_forward_stacked_with_encoder_outputs_equals_forward():
    _, criterion = build(False, False, two_stage=True)
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(6, 2, 300, 91, generator=g)
    boxes = torch.rand(6, 2, 300, 4, generator=g) * 0.5 + 0.25
    enc_logits = torch.randn(2, 747, 91, generator=g)
    enc_boxes = torch.rand(2, 747, 4, generator=g) * 0.5 + 0.25
    targets = [{"boxes": torch.rand(n, 4, generator=g) * 0.4 + 0.3, "labels": torch.randint(0, 90, (n,), generator=g)}
               for n in (5, 9)]
    out = {"pred_logits": logits[-1], "pred_boxes": boxes[-1],
           "aux_outputs": [{"pred_logits": logits[i], "pred_boxes": boxes[i]} for i in range(5)],
           "enc_outputs": {"pred_logits": enc_logits, "pred_boxes": enc_boxes}}
    ref = criterion(out, targets)
    got = criterion.forward_stacked(logits, boxes, targets, enc_outputs=(enc_logits, enc_boxes))
    assert {k for k in ref if k.endswith("_enc")} == {"loss_ce_enc", "loss_bbox_enc", "loss_giou_enc",
                                                     "cardinality_error_enc"}
    for k in ref:
        torch.testing.assert_close(got[k], ref[k], rtol=1e-5, atol=1e-6, msg=k)
