"""The stacked (all-layers-at-once) criterion must reproduce the per-layer loop of the reference
(models/detr.py:382-443) key by key."""
import numpy as np
import pytest
import torch

import set_criterion_fixtures as scf
from conftest import load_golden
from trackformer_b200.model_factory import build_model, default_args


def test_forward_stacked_equals_layer_loop():
    torch.manual_seed(0)
    _, criterion, _ = build_model(default_args(device="cpu", enc_layers=1, dec_layers=6, num_queries=40))
    g = torch.Generator().manual_seed(5)
    k, bs, nq, c = 6, 3, 40, 91
    logits = torch.randn(k, bs, nq, c, generator=g, requires_grad=True)
    boxes_raw = torch.randn(k, bs, nq, 4, generator=g, requires_grad=True)
    boxes = boxes_raw.sigmoid() * 0.5 + 0.2
    targets = []
    for b in range(bs):
        n = 4 + 3 * b
        targets.append({"labels": torch.randint(0, c, (n,), generator=g),
                        "boxes": torch.cat([torch.rand(n, 2, generator=g) * 0.5 + 0.25,
                                            torch.rand(n, 2, generator=g) * 0.3 + 0.05], 1)})
    out = {"pred_logits": logits[-1], "pred_boxes": boxes[-1],
           "aux_outputs": [{"pred_logits": logits[i], "pred_boxes": boxes[i]} for i in range(k - 1)]}
    ref = criterion(out, targets)
    got = criterion.forward_stacked(logits, boxes, targets)
    assert set(ref) == set(got)
    for key in ref:
        torch.testing.assert_close(got[key], ref[key], rtol=1e-5, atol=1e-6, msg=key)
    wd = criterion.weight_dict
    l_ref = sum(ref[key] * wd[key] for key in ref if key in wd)
    l_got = sum(got[key] * wd[key] for key in got if key in wd)
    g_ref = torch.autograd.grad(l_ref, (logits, boxes_raw), retain_graph=True)
    g_got = torch.autograd.grad(l_got, (logits, boxes_raw))
    for a, b in zip(g_got, g_ref):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-7)


@pytest.mark.parametrize("case", ["det", "track"])
def test_forward_stacked_fp64_equals_reference_fixture(case):
    """The host criterion in fp64 (scipy matching, torch losses) against the reference's own SetCriterion on the
    fixture recorded by tests/golden/make_golden_set_criterion.py: same indices, losses and gradients to fp64
    rounding.  The tracking case runs the forced matching (track_queries=True)."""
    from trackformer_b200.criterion import SetCriterion
    from trackformer_b200.matcher import HungarianMatcher
    fx = load_golden("set_criterion", prefix="")
    inp = scf.make_case(case)
    assert scf.checksum(inp) == str(fx[f"{case}_checksum"]), "the fixture's input generator draws differently"
    m = HungarianMatcher(scf.COST_CLASS, scf.COST_BBOX, scf.COST_GIOU, focal_loss=True, focal_alpha=scf.ALPHA,
                         focal_gamma=scf.GAMMA)
    crit = SetCriterion(inp["C"], m, {}, scf.EOS_COEF, ["labels", "boxes", "cardinality"], True, scf.ALPHA,
                        scf.GAMMA, inp["n_track"] > 0, True).double()
    logits = inp["logits"].double().requires_grad_(True)
    boxes = inp["boxes"].double().requires_grad_(True)
    targets = [dict(t, boxes=t["boxes"].double()) for t in inp["targets"]]
    losses = crit.forward_stacked(logits, boxes, targets, track_queries=True)
    ce, l1, gi = losses.stacked
    w = inp["weights"]
    (w[0] * ce + w[1] * l1 + w[2] * gi).sum().backward()
    for key, got in (("loss_ce", ce), ("loss_bbox", l1), ("loss_giou", gi)):
        np.testing.assert_allclose(got.detach().numpy(), fx[f"{case}_{key}"], rtol=1e-12, atol=0, err_msg=key)
    card = torch.stack([losses[f"cardinality_error_{k}"] for k in range(scf.K - 1)] + [losses["cardinality_error"]])
    np.testing.assert_array_equal(card.numpy(), fx[f"{case}_cardinality_error"])
    np.testing.assert_allclose(float(losses["class_error"]), float(fx[f"{case}_class_error"]), rtol=1e-12)
    # matched indices, from the host matcher the criterion used
    layers = [{"pred_logits": logits[k].detach(), "pred_boxes": boxes[k].detach()} for k in range(scf.K)]
    per_layer = m.match_layers_forced(logits.detach(), boxes.detach(), targets) if inp["n_track"] \
        else m.match_layers(layers, targets)
    src, tgt = scf.stacked_indices([[(s.numpy(), t.numpy()) for s, t in layer] for layer in per_layer], inp["sizes"])
    np.testing.assert_array_equal(src, fx[f"{case}_src"])
    np.testing.assert_array_equal(tgt, fx[f"{case}_tgt"])
    # the stored gradients are fp32 roundings of the reference's fp64 ones (the logits' on the stored rows)
    rows = fx[f"{case}_grad_logits_rows"]
    for got, key in ((logits.grad[torch.from_numpy(rows)], "grad_logits"), (boxes.grad, "grad_boxes")):
        ref = fx[f"{case}_{key}"]
        assert np.abs(got.float().numpy() - ref).max() <= 1e-6 * np.abs(ref).max(), key
