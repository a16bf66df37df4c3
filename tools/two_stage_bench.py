#!/usr/bin/env python
"""Two-stage Deformable DETR on the GPU, four comparisons, arms alternated over windows in one process:

  select    the proposal + selection kernels (csrc/two_stage.cu: masking, top-k, gather, reference points, sine
            embedding) against the reference's op chain (gen_encoder_output_proposals without its head, torch.topk,
            gather, sigmoid, get_proposal_pos_embed) at 800x1333, B = 2 (22,223 tokens per image), CUDA-event medians
  match     the encoder matching at S = 22,223, B = 2, T in {20, 100, 300} boxes per image: the workspace Hungarian solver
            (tfb200_lsa_wide_f32) against the cost copy to the host + scipy (host clock, synchronised)
  lsa       the shared-memory solver against the workspace one at Q = 300 (K = 6 layers) and Q = 7,000 (K = 1), the
            workloads on each side of the size choice in the `lsa` binding
  train     the graphed TrainStep (one graph: forward, device matching, loss, backward) at 800x1333, B = 2, 20 boxes per
            image: two-stage against one-stage box refinement, and against the eager reference composition
            (model + SetCriterion.forward + backward, host matching), ms/step

``--check`` compares outputs between the arms (selected tokens and embeddings, matched pairs, losses).  Prints one JSON
line per part with the card name and power limit; stops without a CUDA device.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HW_800 = [(100, 167), (50, 84), (25, 42), (13, 21)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:                                   # noqa: BLE001  (no nvidia-smi: the limit stays unknown)
        return torch.cuda.get_device_name(0), "unknown"


def event_ms(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def host_ms(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def alternate(arms, windows, timer):
    """{name: median ms} over ``windows`` rounds, each round running every arm once in turn"""
    got = {k: [] for k in arms}
    for _ in range(windows):
        for k, fn in arms.items():
            got[k].append(timer(fn))
    return {k: round(statistics.median(v), 4) for k, v in got.items()}


def part_select(dev, args, info):
    from trackformer_b200 import ext
    from trackformer_b200.deformable_transformer import encoder_output_proposals, proposal_dim_t, proposal_pos_embed
    m = ext.load()
    b, k, c = 2, 300, 91
    s = sum(h * w for h, w in HW_800)
    flat = [v for pair in HW_800 for v in pair]
    g = torch.Generator().manual_seed(0)
    memory = torch.randn(b, s, 256, generator=g).to(dev)
    logits = torch.randn(b, s, c, generator=g).to(dev)
    delta = torch.randn(b, s, 4, generator=g).to(dev)
    dim_t = proposal_dim_t(dev)

    def kernels():
        prop, valid, masked = m.two_stage_proposals(None, memory, flat, b, memory.device.index)
        return m.two_stage_select(logits, delta + prop, dim_t, k), masked

    def reference():
        masked, prop = encoder_output_proposals(memory, None, HW_800)
        unact = delta + prop
        idx = torch.topk(logits[..., 0], k, dim=1)[1]
        boxes = torch.gather(unact, 1, idx.unsqueeze(-1).repeat(1, 1, 4)).detach()
        return (idx, boxes, boxes.sigmoid(), proposal_pos_embed(boxes)), masked
    if args.check:
        (ik, bk, rk, ek), mk = kernels()
        (ir, br, rr, er), mr = reference()
        assert torch.equal(ik, ir), "selected tokens differ"
        assert torch.equal(bk, br) and torch.equal(mk, mr)
        info["select_check"] = {"ref_max_abs": float((rk - rr).abs().max()), "embed_max_abs": float((ek - er).abs().max())}
    for fn in (kernels, reference):
        fn()
    info["select_ms"] = alternate({"kernels": kernels, "reference_ops": reference}, args.windows,
                                  lambda fn: event_ms(fn, args.reps))


def part_match(dev, args, info):
    from scipy.optimize import linear_sum_assignment
    from trackformer_b200 import ext
    m = ext.load()
    b, s, c = 2, sum(h * w for h, w in HW_800), 91
    g = torch.Generator().manual_seed(1)
    logits = torch.randn(1, b, s, c, generator=g).to(dev)
    boxes = (torch.rand(1, b, s, 4, generator=g) * 0.8 + 0.1).to(dev)
    out = {}
    for t in args.targets:
        tgt_boxes = torch.cat([torch.rand(b * t, 2, generator=g) * 0.6 + 0.2, torch.rand(b * t, 2, generator=g) * 0.2 + 0.05],
                              1).to(dev)
        tgt_ids = torch.zeros(b * t, dtype=torch.int64, device=dev)
        cost = m.match_cost(logits, boxes, tgt_ids, tgt_boxes, 2.0, 5.0, 2.0, 0.25, 2.0).view(1, b, s, b * t)
        off = torch.tensor([0, t, 2 * t], dtype=torch.int32, device=dev)

        def device():
            return m.lsa(cost, off, t)

        def host():
            c_host = cost.cpu()
            return [linear_sum_assignment(c_host[0, i, :, i * t:(i + 1) * t]) for i in range(b)]
        if args.check:
            src, tgt, status = device()
            assert int(status) == 0
            for i, (r, cc) in enumerate(host()):
                order = np.argsort(r)
                assert np.array_equal(src[0, i * t:(i + 1) * t].cpu().numpy(), r[order])
                assert np.array_equal(tgt[0, i * t:(i + 1) * t].cpu().numpy() - i * t, cc[order])
        device()
        out[t] = alternate({"wide_kernel": device, "copy_scipy": host}, args.windows, lambda fn: host_ms(fn, 3))
    info["match_ms"] = out


def part_lsa(dev, args, info):
    from trackformer_b200 import ext
    m = ext.load()
    out = {}
    for q, k, t in ((300, 6, 100), (7000, 1, 100)):
        g = torch.Generator().manual_seed(q)
        cost = (torch.rand(k, 2, q, 2 * t, generator=g) * 10).to(dev)
        off = torch.tensor([0, t, 2 * t], dtype=torch.int32, device=dev)
        shared, wide = m.lsa(cost, off, t), m.lsa_wide(cost, off, t)
        if args.check:
            assert all(torch.equal(x, y) for x, y in zip(shared, wide)), f"solvers differ at Q={q}"
        out[q] = alternate({"shared_memory": lambda: m.lsa(cost, off, t), "workspace": lambda: m.lsa_wide(cost, off, t)},
                           args.windows, lambda fn: event_ms(fn, args.reps))
    info["lsa_ms"] = out


def part_train(dev, args, info):
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.train_step import TrainStep
    g = torch.Generator().manual_seed(2)
    frames = torch.randn(2, 3, 800, 1333, generator=g).to(dev)

    def targets():
        return [{"boxes": torch.cat([torch.rand(20, 2, generator=g) * 0.6 + 0.2, torch.rand(20, 2, generator=g) * 0.2 + 0.05],
                                    1).to(dev), "labels": torch.zeros(20, dtype=torch.int64, device=dev)} for _ in range(2)]
    tg = targets()
    arms = {}
    models = {}
    for name, two_stage in (("two_stage", True), ("one_stage", False)):
        torch.manual_seed(0)
        model, criterion, _ = build_model(default_args(device=str(dev), dropout=0.0, two_stage=two_stage))
        model.to(dev).train()
        models[name] = (copy.deepcopy(model) if two_stage else None, criterion)
        step = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames, example_targets=tg)
        assert step.g_full is not None
        arms[name] = (lambda s: (lambda: s(frames, tg)))(step)
    ref_model, ref_crit = models["two_stage"]

    def eager():
        ref_model.zero_grad(set_to_none=True)
        out = ref_model(frames, tg)[0]
        loss_dict = ref_crit(out, tg)
        loss = sum(loss_dict[k] * ref_crit.weight_dict[k] for k in loss_dict if k in ref_crit.weight_dict)
        loss.backward()
        return loss
    arms["two_stage_eager_reference"] = eager
    for fn in arms.values():
        fn()
    if args.check:
        a, b = float(arms["two_stage"]()), float(eager())
        info["train_check"] = {"graphed_loss": a, "eager_loss": b, "rel": abs(a - b) / abs(b)}
    info["train_ms_per_step"] = alternate(arms, args.windows, lambda fn: host_ms(fn, args.train_steps))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--parts", nargs="+", default=["select", "match", "lsa", "train"])
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--train-steps", type=int, default=5)
    ap.add_argument("--targets", type=int, nargs="+", default=[20, 100, 300])
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("two_stage_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    for part in args.parts:
        info = {"part": part, "card": name, "power_limit": power, "windows": args.windows,
                "tf32": torch.backends.cuda.matmul.allow_tf32}
        {"select": part_select, "match": part_match, "lsa": part_lsa, "train": part_train}[part](dev, args, info)
        print(json.dumps(info), flush=True)


if __name__ == "__main__":
    main()
