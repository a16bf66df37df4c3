"""CPU tests of the segmentation models (trackformer_b200/segmentation.py), the ``masks`` loss and the factory.

The CPU path of the mask head runs the reference's torch ops; these tests check the model surface (class layout,
parameter names and shapes of src/trackformer/models/detr_segmentation.py), the loss against a literal restatement of
the reference's loss_masks (models/detr.py:330-357), and argument validation of the new C entry points.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import model_fixtures as mf

MASK_KEYS = ({f"bbox_attention.{m}_linear.{p}" for m in "qk" for p in ("weight", "bias")}
             | {f"mask_head.{m}.{p}" for m in ("lay1", "lay2", "lay3", "lay4", "lay5", "gn1", "gn2", "gn3", "gn4",
                                                 "gn5", "out_lay", "adapter1", "adapter2", "adapter3")
                for p in ("weight", "bias")})


@pytest.fixture()
def oracle_op(monkeypatch):
    """The product has no CPU path for the MSDeformAttn core: the forward test substitutes the oracle's torch
    restatement for it, as tests/test_model_parity_cpu.py does."""
    from oracle.torch_ref import msda_core_torch
    import trackformer_b200.msda_module as mm

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    monkeypatch.setattr(mm, "MSDeformAttnFunction", _OracleFn)


def _build(tracking=False, **overrides):
    from trackformer_b200.model_factory import build_model, default_args
    torch.manual_seed(0)
    return build_model(default_args(tracking, device="cpu", masks=True, **overrides))


def test_state_dict_names_and_shapes_match_reference_layout():
    from trackformer_b200.model_factory import build_model, default_args
    torch.manual_seed(0)
    base, _, _ = build_model(default_args(device="cpu"))
    model, _, _ = _build()
    keys, base_keys = set(model.state_dict()), set(base.state_dict())
    assert base_keys <= keys and keys - base_keys == MASK_KEYS
    sd = model.state_dict()
    expect = {"mask_head.lay1.weight": (264, 264, 3, 3), "mask_head.gn1.weight": (264,),
              "mask_head.lay2.weight": (128, 264, 3, 3), "mask_head.lay5.weight": (16, 32, 3, 3),
              "mask_head.out_lay.weight": (1, 16, 3, 3), "mask_head.adapter1.weight": (128, 1024, 1, 1),
              "mask_head.adapter2.weight": (64, 512, 1, 1), "mask_head.adapter3.weight": (32, 256, 1, 1),
              "bbox_attention.k_linear.weight": (256, 256)}
    for k, shape in expect.items():
        assert tuple(sd[k].shape) == shape, k


def test_factory_builds_segmentation_models():
    from trackformer_b200.detr_tracking import DETRTrackingBase
    from trackformer_b200.deformable_detr import DeformableDETR
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.segmentation import (DETRSegmBase, DeformableDETRSegm, DeformableDETRSegmTracking,
                                               PostProcessSegm)
    model, criterion, post = _build()
    assert type(model) is DeformableDETRSegm
    assert "masks" in criterion.losses and isinstance(post["segm"], PostProcessSegm)
    assert criterion.weight_dict["loss_mask"] == 1.0 and criterion.weight_dict["loss_dice"] == 1.0
    assert "loss_mask_0" in criterion.weight_dict                    # the reference's aux weight copy (__init__.py:92-98)
    model, _, _ = _build(tracking=True)
    assert type(model) is DeformableDETRSegmTracking
    mro = type(model).__mro__
    assert mro.index(DETRSegmBase) < mro.index(DETRTrackingBase) < mro.index(DeformableDETR)
    frozen, _, _ = _build(freeze_detr=True)
    trainable = {n for n, p in frozen.named_parameters() if p.requires_grad}
    assert trainable == {k for k in MASK_KEYS}
    with pytest.raises(NotImplementedError, match="panoptic"):
        build_model(default_args(device="cpu", masks=True, dataset="coco_panoptic"))


def test_cpu_forward_shapes_and_prev_features(oracle_op):
    model, _, _ = _build(tracking=True)
    mf.canonical_weights_(model, 0)
    model.tracking()
    f1, f2 = mf.make_images(3, [(160, 224), (160, 224)])
    with torch.no_grad():
        out1, _, feats1, _, _ = model(f1[None])                           # the two-argument call keeps working
        tgt = [{"track_query_boxes": out1["pred_boxes"][0, :4], "track_query_hs_embeds": out1["hs_embed"][0, :4],
                "image_id": torch.tensor([1])}]
        out2, _, _, _, _ = model(f2[None], tgt, feats1)                  # the tracker's three-argument call
    assert out1["pred_masks"].shape == (1, 300, 40, 56)
    assert out2["pred_masks"].shape == (1, 304, 40, 56)
    assert torch.isfinite(out2["pred_masks"]).all()


def _targets_with_masks(seed, sizes, n_boxes):
    g = torch.Generator().manual_seed(seed)
    out = mf.make_targets(seed, len(sizes), 0)
    for t, (h, w), n in zip(out, sizes, n_boxes):
        t["masks"] = torch.rand(n, h, w, generator=g) > 0.6
        t["labels"] = torch.zeros(n, dtype=torch.int64)
    return out


def reference_loss_masks(pred_masks, targets, indices, num_boxes):
    """detr.py:330-357 restated with util/misc.py's nested_tensor_from_tensor_list, sigmoid_focal_loss, dice_loss."""
    masks = [t["masks"] for t in targets]
    n, h, w = (max(m.shape[i] for m in masks) for i in range(3))
    tm = torch.zeros(len(masks), n, h, w, dtype=pred_masks.dtype)
    for b, m in enumerate(masks):
        tm[b, :m.shape[0], :m.shape[1], :m.shape[2]] = m.to(tm)
    bi = torch.cat([torch.full_like(s, b) for b, (s, _) in enumerate(indices)])
    si = torch.cat([s for s, _ in indices])
    ti = torch.cat([t for _, t in indices])
    src = F.interpolate(pred_masks[bi, si][:, None], size=(h, w), mode="bilinear", align_corners=False)[:, 0].flatten(1)
    tgt = tm[bi, ti].flatten(1)
    prob = src.sigmoid()
    ce = F.binary_cross_entropy_with_logits(src, tgt, reduction="none")
    p_t = prob * tgt + (1 - prob) * (1 - tgt)
    focal = (0.25 * tgt + 0.75 * (1 - tgt)) * ce * (1 - p_t) ** 2
    dice = 1 - (2 * (prob * tgt).sum(1) + 1) / (prob.sum(-1) + tgt.sum(-1) + 1)
    return focal.mean(1).sum() / num_boxes, dice.sum() / num_boxes


def test_loss_masks_matches_reference_restatement():
    _, criterion, _ = _build()
    g = torch.Generator().manual_seed(1)
    pred = torch.randn(2, 12, 10, 14, generator=g, dtype=torch.float64, requires_grad=True)
    targets = _targets_with_masks(2, [(37, 50), (40, 45)], [3, 2])
    indices = [(torch.tensor([4, 0, 9]), torch.tensor([2, 0, 1])), (torch.tensor([11, 3]), torch.tensor([1, 0]))]
    got = criterion.loss_masks({"pred_masks": pred}, targets, indices, 4.0)
    ref = reference_loss_masks(pred, targets, indices, 4.0)
    torch.testing.assert_close(got["loss_mask"], ref[0], rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(got["loss_dice"], ref[1], rtol=1e-12, atol=1e-14)
    empty = [(torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64))] * 2
    zero = criterion.loss_masks({"pred_masks": pred}, targets, empty, 1.0)
    assert float(zero["loss_mask"]) == 0.0 and float(zero["loss_dice"]) == 0.0


def test_forward_stacked_adds_mask_losses_of_the_last_layer():
    _, criterion, _ = _build()
    g = torch.Generator().manual_seed(3)
    k, b, q = 6, 2, 300
    logits = torch.randn(k, b, q, 91, generator=g)
    boxes = torch.rand(k, b, q, 4, generator=g) * 0.5 + 0.25
    pred_masks = torch.randn(b, q, 10, 14, generator=g)
    targets = _targets_with_masks(4, [(40, 56), (36, 50)], [3, 2])
    for t in targets:
        t["boxes"] = torch.rand(len(t["masks"]), 4, generator=g) * 0.4 + 0.3
    stacked = criterion.forward_stacked(logits, boxes, targets, pred_masks=pred_masks)
    out = {"pred_logits": logits[-1], "pred_boxes": boxes[-1], "pred_masks": pred_masks,
           "aux_outputs": [{"pred_logits": logits[i], "pred_boxes": boxes[i]} for i in range(k - 1)]}
    eager = criterion(out, targets)
    assert stacked.stacked is not None                                   # the stacked route, not the per-layer fallback
    for key in ("loss_mask", "loss_dice", "loss_ce", "loss_bbox"):
        torch.testing.assert_close(stacked[key], eager[key], rtol=1e-5, atol=1e-6)
    assert "loss_mask_0" not in eager


def test_train_step_rejects_mask_models():
    from trackformer_b200.train_step import TrainStep
    model, criterion, _ = _build()
    with pytest.raises(NotImplementedError, match="segmentation"):
        TrainStep(model, criterion, use_graphs=False)


def test_mask_head_entry_points_validate_arguments():
    from trackformer_b200 import _build as b
    lib = ctypes.CDLL(b.build_library())
    vp, i, i64, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, vp)
    attn = lib.tfb200_mask_attn_fwd_f32
    attn.argtypes = [vp, vp, vp, vp, i, i, i, i, f, vp]
    assert attn(None, p, None, p, 1, 1, 4, 8, 1.0, None) == -1
    assert attn(p, p, None, p, 1, 1, 0, 8, 1.0, None) == -2
    assert attn(p, p, None, p, 0, 5, 4, 8, 1.0, None) == 0                # empty batch is a no-op
    odd = ctypes.c_void_p(ctypes.addressof(buf) + 4)
    assert attn(odd, p, None, p, 1, 1, 4, 8, 1.0, None) == -2            # q not 16-byte aligned
    assert attn(p, odd, None, p, 1, 1, 4, 8, 1.0, None) == -2            # k not 16-byte aligned
    attn_bwd = lib.tfb200_mask_attn_bwd_f32
    attn_bwd.argtypes = [vp] * 7 + [i, i, i, i, f, vp]
    assert attn_bwd(p, p, p, p, p, p, odd, 1, 1, 4, 8, 1.0, None) == -2  # dk not 16-byte aligned
    gn = lib.tfb200_group_norm_relu_fwd_f32
    gn.argtypes = [vp] * 7 + [i, i, i64, i, i, f, vp]
    assert gn(p, None, p, p, p, p, None, 2, 1, 16, 16, 8, 1e-5, None) == -1          # no rstd
    assert gn(p, None, p, p, p, p, p, 2, 1, 16, 18, 8, 1e-5, None) == -2             # C % groups
    assert gn(p, None, p, p, p, p, p, 3, 2, 16, 16, 8, 1e-5, None) == -2             # N % per_image
    assert gn(p, None, p, p, p, p, p, 2, 1, 16, 8 * 264, 8, 1e-5, None) == -2        # > 256 channels per group
    up = lib.tfb200_upsample_add_fwd_f32
    up.argtypes = [vp, vp, vp] + [i] * 7 + [vp]
    assert up(p, None, p, 2, 1, 4, 4, 8, 8, 16, None) == -1
    assert up(p, p, p, 2, 1, 0, 4, 8, 8, 16, None) == -2
    loss = lib.tfb200_mask_loss_fwd_f32
    loss.argtypes = [vp] * 8 + [i] * 5 + [f, f, vp]
    assert loss(p, p, p, p, p, p, p, p, -1, 4, 4, 8, 8, 0.25, 2.0, None) == -2
    assert loss(p, None, p, p, p, p, p, p, 3, 4, 4, 8, 8, 0.25, 2.0, None) == -1
    assert loss(p, p, p, p, p, p, p, p, 3, 0, 4, 8, 8, 0.25, 2.0, None) == -2


def test_python_bindings_reject_cpu_tensors():
    from trackformer_b200 import ext
    m = ext.load()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.mask_attn_forward(torch.zeros(1, 2, 256), torch.zeros(1, 4, 256), None, 8, 1.0)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.group_norm_relu_forward(torch.zeros(2, 16, 4, 4), None, torch.ones(16), torch.zeros(16), 8, 1, 1e-5)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.upsample_add_forward(torch.zeros(2, 16, 4, 4), torch.zeros(1, 16, 8, 8))
