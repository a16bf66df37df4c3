"""The vanilla-DETR family on CPU (DETR, DETRTracking, DETRSegm, DETRSegmTracking, PostProcess, the ``deformable=False``
route of build_model) against fixtures recorded from the reference's own classes (tests/golden/make_golden_detr.py)."""
import numpy as np
import pytest
import torch

import detr_fixtures as df
from conftest import load_golden


@pytest.mark.parametrize("case", ["det_mini", "det_padded_batch", "track_two_frames", "segm_track_two_frames"])
def test_forward_matches_reference(case):
    df.check(df.run_case(case), load_golden(case, "detr_"), rtol=1e-4, rel_atol=1e-4)


@pytest.mark.parametrize("case", ["train_step_det", "train_step_tracking", "segm_det_mini"])
def test_train_step_losses_and_gradients_match_reference(case):
    df.check(df.run_case(case), load_golden(case, "detr_"), rtol=1e-3, rel_atol=1e-4)


def test_state_dicts_equal_the_reference():
    from trackformer_b200.model_factory import build_model, vanilla_args
    gold = load_golden("state_dicts", "detr_")
    for name, tracking, masks in (("DETR", False, False), ("DETRTracking", True, False),
                                  ("DETRSegm", False, True), ("DETRSegmTracking", True, True)):
        model, _ = df.build(tracking, False, masks=masks)
        assert type(model).__name__ == name
        assert df.state_dict_layout(model) == df.recorded_layout(gold, name), name
    model, _, post = build_model(vanilla_args(tracking=True, masks=True, dataset="mot", device="cpu"))
    assert type(model).__name__ == "DETRSegmTracking"
    assert df.state_dict_layout(model) == df.recorded_layout(gold, "DETRSegmTracking")
    assert "transformer.decoder.layers.5.multihead_attn.in_proj_weight" in model.state_dict()


def test_factory_routes_and_vanilla_args():
    from trackformer_b200.deformable_detr import DeformablePostProcess, PostProcess
    from trackformer_b200.model_factory import build_model, default_args, vanilla_args
    a = vanilla_args()
    assert not a.deformable and not a.focal_loss and a.num_queries == 100 and a.dim_feedforward == 2048
    assert not a.tracking and not a.masks and a.dataset == "coco"
    t = vanilla_args(tracking=True, masks=True, dataset="mot")
    assert t.tracking and t.track_prev_frame_range == 5 and t.track_query_false_positive_eos_weight and t.masks
    assert default_args().deformable                          # unchanged meaning
    torch.manual_seed(0)
    model, crit, post = build_model(vanilla_args(device="cpu", enc_layers=1, dec_layers=2))
    assert type(model).__name__ == "DETR" and isinstance(post["bbox"], PostProcess) and not crit.focal_loss
    assert crit.num_classes == 91 and model.class_embed.out_features == 92
    assert "loss_ce_0" in crit.weight_dict and "loss_ce_1" not in crit.weight_dict
    _, _, post = build_model(default_args(device="cpu", enc_layers=1, dec_layers=1))
    assert isinstance(post["bbox"], DeformablePostProcess)
    model, _, post = build_model(vanilla_args(tracking=True, masks=True, dataset="mot", device="cpu", enc_layers=1,
                                              dec_layers=1))
    assert type(model).__name__ == "DETRSegmTracking" and "segm" in post


def test_track_attention_is_rejected():
    from trackformer_b200.model_factory import build_model, vanilla_args
    with pytest.raises(NotImplementedError, match="track_attention"):
        build_model(vanilla_args(device="cpu", track_attention=True))


def test_postprocess_matches_reference():
    from trackformer_b200.deformable_detr import PostProcess
    gold = load_golden("postprocess", "detr_")
    outputs = {"pred_logits": torch.from_numpy(gold["logits"]), "pred_boxes": torch.from_numpy(gold["boxes"])}
    sizes = torch.from_numpy(gold["sizes"])
    res = PostProcess()(outputs, sizes)
    for i, r in enumerate(res):
        for k, v in r.items():
            np.testing.assert_allclose(v.numpy(), gold[f"{i}/{k}"], rtol=1e-6, atol=1e-6, err_msg=f"{i}/{k}")
    rows = PostProcess().packed(outputs, sizes)
    for i in range(len(res)):
        np.testing.assert_allclose(rows[i, :, 0].numpy(), gold[f"{i}/scores"], rtol=1e-6)
        np.testing.assert_array_equal(rows[i, :, 1].numpy(), gold[f"{i}/labels"].astype(np.float32))
        np.testing.assert_array_equal(rows._labels[i].numpy(), gold[f"{i}/labels"])
        np.testing.assert_allclose(rows[i, :, 2:].numpy(), gold[f"{i}/boxes"], rtol=1e-6, atol=1e-4)
    assert gold["0/labels"][3] == 2                             # the recorded tie went to the smaller class index


def test_prev_features_is_accepted_and_ignored():
    model, _ = df.build(True, False, enc_layers=1, dec_layers=1)
    model.tracking()
    img = torch.randn(1, 3, 96, 128, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        a = model(img)
        b = model(img, None, a[2])
    torch.testing.assert_close(a[0]["pred_logits"], b[0]["pred_logits"], rtol=0, atol=0)
