#!/usr/bin/env python
"""Softmax set-criterion golden fixture recorded FROM THE REFERENCE (runs on the CPU).

Runs the reference's own HungarianMatcher (models/matcher.py) and SetCriterion (models/detr.py:139-443) with the
softmax classifier of cfgs/train.yaml (``focal_loss: false``, ``eos_coef`` 0.1, ``tracking: true``) and 5 auxiliary
layers, on CPU in fp64, imported as tests/golden/make_golden_model.py imports the reference, on the inputs of
tests/softmax_criterion_fixtures.py (C + 1 = 92 and 21, 100 object queries behind pinned and false-positive track
queries), once with ``track_query_false_positive_eos_weight`` on ("fp1") and once off ("fp0").  Stores
tests/golden/softmax_criterion.npz with, per case and setting (prefix ``<case>_<fp>_``):

  loss_ce, loss_bbox, loss_giou, cardinality_error [K]   layer k < K-1 is aux layer k, K-1 the last layer
  class_error                                            the last layer's
  src, tgt [K, T]                                        matched query / global box per layer, images in order
  grad_boxes [K,B,Q,4] (fp32)                            gradient of sum_k w[0,k] loss_ce_k + w[1,k] loss_bbox_k
                                                         + w[2,k] loss_giou_k with the fixture's seeded weights
  grad_logits_rows [K,B,Q] (bool)                        every row of the last layer and every matched row
  grad_logits [rows, C+1] (fp32)                         the logit gradient of the same total on those rows
  checksum                                               SHA-256 of the regenerated inputs

Before saving, the script asserts that scipy picks the same indices on the reference's fp64 cost, on the cost the
reference computes in fp32, and on the fp64 cost under 1e-5 relative noise.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE)))

import softmax_criterion_fixtures as smf  # noqa: E402


def _outputs(logits, boxes):
    return {"pred_logits": logits[-1], "pred_boxes": boxes[-1],
            "aux_outputs": [{"pred_logits": logits[k], "pred_boxes": boxes[k]} for k in range(smf.K - 1)]}


def _targets(case, dtype):
    return [{k: (v.to(dtype) if k == "boxes" else v) for k, v in t.items()} for t in case["targets"]]


def run_case(name, fp, ref_matcher, SetCriterion):
    case = smf.make_case(name)
    C, sizes = case["C"], case["sizes"]
    matcher = ref_matcher.HungarianMatcher(cost_class=smf.COST_CLASS, cost_bbox=smf.COST_BBOX,
                                           cost_giou=smf.COST_GIOU, focal_loss=False)
    crit = SetCriterion(C - 1, matcher=matcher, weight_dict={}, eos_coef=smf.EOS_COEF,
                        losses=["labels", "boxes", "cardinality"], focal_loss=False, focal_alpha=0.25,
                        focal_gamma=2.0, tracking=True, track_query_false_positive_eos_weight=smf.FP_WEIGHT[fp])

    seen = []
    real_lsa = ref_matcher.linear_sum_assignment

    def spy(c):
        r = real_lsa(c)
        seen.append((np.array(c, dtype=np.float64), r))
        return r
    ref_matcher.linear_sum_assignment = spy
    try:
        logits = case["logits"].double().requires_grad_(True)
        boxes = case["boxes"].double().requires_grad_(True)
        crit.empty_weight = crit.empty_weight.double()
        losses = crit(_outputs(logits, boxes), _targets(case, torch.float64))
        f64 = list(seen)
        seen.clear()
        crit.empty_weight = crit.empty_weight.float()
        with torch.no_grad():
            crit(_outputs(case["logits"], case["boxes"]), _targets(case, torch.float32))
        f32 = list(seen)
    finally:
        ref_matcher.linear_sum_assignment = real_lsa

    g = np.random.default_rng(7)
    assert len(f64) == len(f32) == smf.K * len(sizes)
    for (c64, r64), (_, r32) in zip(f64, f32):
        noisy = c64 * (1 + 1e-5 * g.uniform(-1, 1, c64.shape))
        rn = real_lsa(noisy)
        for r in (r32, rn):
            assert np.array_equal(r[0], r64[0]) and np.array_equal(r[1], r64[1]), name

    # matcher calls run last layer first, then aux 0..K-2; one call per image each
    B = len(sizes)
    per_call = [[(r[0], r[1]) for _, r in f64[i * B:(i + 1) * B]] for i in range(smf.K)]
    per_layer = per_call[1:] + per_call[:1]
    src, tgt = smf.stacked_indices(per_layer, sizes)

    def key(base, k):
        return base if k == smf.K - 1 else f"{base}_{k}"
    res = {}
    for base in ("loss_ce", "loss_bbox", "loss_giou", "cardinality_error"):
        res[base] = np.array([float(losses[key(base, k)]) for k in range(smf.K)])
    res["class_error"] = np.array(float(losses["class_error"]))
    w = case["weights"]
    total = sum(w[i, k] * losses[key(base, k)] for i, base in enumerate(("loss_ce", "loss_bbox", "loss_giou"))
                for k in range(smf.K))
    total.backward()
    rows = smf.grad_logits_rows(src, tgt, sizes, logits.shape[2])
    res.update(src=src, tgt=tgt, grad_logits_rows=rows, grad_logits=logits.grad.float().numpy()[rows],
               grad_boxes=boxes.grad.float().numpy(), checksum=np.array(smf.checksum(case)))
    print(f"{name} {fp}: loss_ce {res['loss_ce'][-1]:.5f} loss_bbox {res['loss_bbox'][-1]:.4f} "
          f"loss_giou {res['loss_giou'][-1]:.4f} class_error {float(res['class_error']):.2f}", flush=True)
    return {f"{name}_{fp}_{k}": v for k, v in res.items()}


def main():
    from make_golden_model import import_reference
    import_reference()
    import trackformer.models.matcher as ref_matcher
    from trackformer.models.detr import SetCriterion
    res = {}
    for name in smf.CASES:
        for fp in smf.FP_WEIGHT:
            res.update(run_case(name, fp, ref_matcher, SetCriterion))
    path = os.path.join(HERE, "softmax_criterion.npz")
    np.savez_compressed(path, **res)
    print(f"softmax_criterion -> {os.path.relpath(path)} ({os.path.getsize(path) / 1024:.0f} KiB)", flush=True)


if __name__ == "__main__":
    main()
