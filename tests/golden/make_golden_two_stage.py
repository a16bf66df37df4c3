#!/usr/bin/env python
"""Two-stage Deformable DETR golden fixtures recorded FROM THE REFERENCE (build container only).

The reference's classes run on the CPU as in make_golden_model.py (canonical weights, the pure-PyTorch MSDeformAttn),
driven by the runners of tests/two_stage_fixtures.py, with ``two_stage: true`` on top of train_deformable.yaml.  Hooks on
the reference transformer also record the padding mask and the level sizes, the proposal logits of every token, the
gathered unactivated boxes of the selected tokens and rows of their sine embedding.  Output:
tests/golden/two_stage_<case>.npz.
"""
import os
import sys

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
REF = "/root/reference"
EMBED_ROWS = 16
MIN_BOUNDARY_GAP = 1e-3


def probe(model):
    tr = model.transformer
    seen = {}
    gen, embed = tr.gen_encoder_output_proposals, tr.get_proposal_pos_embed

    def gen_hook(memory, mask, shapes):
        out_memory, proposals = gen(memory, mask, shapes)
        seen["mask"] = mask.detach().to(torch.uint8).numpy().copy()
        seen["hw"] = shapes.detach().numpy().astype(np.int32).copy()
        seen["prop"] = proposals.detach().numpy().copy()
        return out_memory, proposals

    def embed_hook(proposals):
        pos = embed(proposals)
        seen["topk_unact"] = proposals.detach().numpy().copy()
        seen["embed_rows"] = pos[:, :EMBED_ROWS].detach().numpy().copy()
        return pos
    tr.gen_encoder_output_proposals = gen_hook
    tr.get_proposal_pos_embed = embed_hook
    return lambda: dict(seen)


def main():
    import two_stage_fixtures as tf
    from make_golden_model import import_reference
    build_model, to_ns = import_reference()

    def load(name):
        return yaml.safe_load(open(os.path.join(REF, "cfgs", name)))

    def build(tracking, multi_frame, **overrides):
        assert not tracking and not multi_frame
        cfg = load("train.yaml")
        cfg.update(load("train_deformable.yaml"))
        cfg["device"] = "cpu"
        cfg.update(overrides)
        torch.manual_seed(0)
        model, criterion, _ = build_model(to_ns(cfg))
        return model, criterion

    cases = {
        "det_mini": lambda: tf.run_detection(build, [(160, 224)], probe=probe),
        "det_padded_batch": lambda: tf.run_detection(build, [(160, 224), (128, 192)], seed=1, probe=probe),
        "det_800x1333": lambda: tf.run_detection(build, [(800, 1333)], seed=1, probe=probe),
        "train_step_det": lambda: tf.run_train_step(build, [(160, 224), (160, 224)], 6, seed=tf.TRAIN_STEP_SEED,
                                                    probe=probe),
        "segm_det_mini": lambda: tf.run_detection(build, [(160, 224)], masks=True, probe=probe),
    }
    only = sys.argv[1:]
    for name, fn in cases.items():
        if only and name not in only:
            continue
        res = fn()
        # seeds are chosen so that no selection sits within 1e-3 of a tie at the k-th logit
        assert res["boundary_gap"].min() >= MIN_BOUNDARY_GAP, (name, res["boundary_gap"])
        path = os.path.join(HERE, f"two_stage_{name}.npz")
        np.savez_compressed(path, **{k: np.asarray(v) for k, v in res.items()})
        gap = res.get("boundary_gap")
        print(f"{name:18s} -> {os.path.relpath(path)} ({os.path.getsize(path) / 1024:.0f} KiB), boundary gap "
              f"{None if gap is None else gap.min():.3g}, min adjacent gap {res['min_adjacent_gap'].min():.3g}",
              flush=True)
    if not only or "state_dict" in only:
        model, _ = build(False, False, two_stage=True)
        path = os.path.join(HERE, "two_stage_state_dict.npz")
        np.savez_compressed(path, **tf.state_dict_shapes(model))
        print(f"state_dict         -> {os.path.relpath(path)}")


if __name__ == "__main__":
    main()
