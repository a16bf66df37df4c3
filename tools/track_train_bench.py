#!/usr/bin/env python
"""Tracking training step on one GPU: the eager reference composition against TrainStep's tracking route.

Workload: the tracking model (deformable DETR R50, 20-class head, random-init weights) trained on two-frame samples of
`--height` x `--width` (default 800x1333, the geometry of BASELINE.json configs[2]) with 300 object queries, or with
`--multi-frame` the documented training model (default_args(tracking=True, multi_frame=True): 500 queries, hidden 288,
multi-frame attention, 8 levels), or with `--vanilla` the vanilla-DETR tracking model (vanilla_args(tracking=True):
cfgs/train.yaml + train_tracking.yaml, 100 object queries, dense attention, a 21-class softmax head, whose
SetCriterion is the weighted cross-entropy one).  Synthetic previous / current targets carry `--boxes` boxes per frame with shared
identities, so the previous frame's matching keeps enough identities for about `--tracks` track queries; the CPU
generator is re-seeded before every step with a seed whose first two bookkeeping draws (detr_tracking.py: how many
matches survive, how many false positives) give that count, so every timed step has the same K.

Arms, alternated in the same run, each timed as ms/step with a device synchronise at the end of the timed window:
  eager   model(samples, targets) + SetCriterion + backward + clip_grad_norm_ + torch.optim.AdamW (reference groups)
  graphed TrainStep(track_bucket=--bucket, flat_adamw=reference groups): previous frame from a graph, device matching,
          bookkeeping, padded current frame from forward / backward graphs, forced device matching + fused loss,
          one-pass clip + AdamW

`--masks` trains the segmentation variant of the chosen model (DeformableDETRSegmTracking, or DETRSegmTracking with
`--vanilla`): the targets carry one mask per box, the eager arm runs the reference's all-row mask head, the graphed arm
is TrainStep(masks=True), whose mask head runs on the matched rows only.  Every arm also reports its peak allocated
memory over its timed windows (torch.cuda.max_memory_allocated, both models' weights and optimiser state included).

`--check` (dropout 0): before timing, both arms take the same seeded step from the same weights; their track-query
indices must be equal and their loss and a seeded gradient sample close.

Prints one JSON line with the card name and power limit; tools/README.md lists it among the measurement aids.
"""
import argparse
import copy
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:                                   # noqa: BLE001  (no nvidia-smi: the limit stays unknown)
        return torch.cuda.get_device_name(0), "unknown"


def make_sample(g, dev, size, n_boxes, batch, masks=False):
    """current frame + targets with prev_image / prev_target; the previous frame drops 5 identities and has 5 new ones;
    with ``masks`` every box of the current frame gets a mask (its interior, ragged)"""
    h, w = size
    frames = torch.randn(batch, 3, h, w, generator=g).to(dev)
    targets = []
    for _ in range(batch):
        cxcy = torch.rand(n_boxes, 2, generator=g) * 0.8 + 0.1
        wh = torch.rand(n_boxes, 2, generator=g) * 0.06 + 0.02
        boxes = torch.cat([cxcy, wh], 1)
        ids = torch.arange(n_boxes)
        prev_ids = torch.cat([ids[5:], torch.arange(1000, 1005)])
        prev_boxes = (boxes + (torch.rand(n_boxes, 4, generator=g) - 0.5) * 0.01).clamp(0.01, 0.99)
        t = {"boxes": boxes, "labels": torch.zeros(n_boxes, dtype=torch.int64), "track_ids": ids,
             "image_id": torch.tensor([0])}
        pt = {"boxes": prev_boxes, "labels": torch.zeros(n_boxes, dtype=torch.int64), "track_ids": prev_ids,
              "image_id": torch.tensor([0])}
        if masks:
            ys = torch.arange(h, dtype=torch.float32)[:, None] / h
            xs = torch.arange(w, dtype=torch.float32)[None, :] / w
            t["masks"] = torch.stack([((xs - cx).abs() <= bw / 2) & ((ys - cy).abs() <= bh / 2)
                                      & (torch.rand(h, w, generator=g) > 0.1)
                                      for cx, cy, bw, bh in boxes.tolist()])
        t = {k: v.to(dev) for k, v in t.items()}
        t["prev_target"] = {k: v.to(dev) for k, v in pt.items()}
        t["prev_image"] = torch.randn(3, h, w, generator=g).to(dev)
        targets.append(t)
    return frames, targets


def seed_for(n_track, n_matched, fp_prob):
    """a seed whose first two draws of add_track_queries_to_targets keep about n_track track queries"""
    best = (None, -1)
    for seed in range(10000):
        torch.manual_seed(seed)
        keep = torch.randint(0, n_matched + 1, (1,)).item()
        fp = torch.randint(int(math.ceil(fp_prob * keep)) + 1, (1,)).item() if keep else 0
        if abs(keep + fp - n_track) < abs(best[1] - n_track):
            best = (seed, keep + fp)
        if keep + fp == n_track:
            break
    return best[0]


def fresh(targets):
    """the bookkeeping writes into the target dicts: every step gets its own"""
    return [dict(t) for t in targets]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the two arms")
    ap.add_argument("--height", type=int, default=800)
    ap.add_argument("--width", type=int, default=1333)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--boxes", type=int, default=None, help="boxes per frame (default 120; 60 with --vanilla)")
    ap.add_argument("--tracks", type=int, default=None, help="track queries (default 100; 50 with --vanilla)")
    ap.add_argument("--bucket", type=int, default=32)
    ap.add_argument("--multi-frame", action="store_true")
    ap.add_argument("--vanilla", action="store_true", help="vanilla-DETR tracking model (softmax classifier)")
    ap.add_argument("--masks", action="store_true", help="the segmentation model (TrainStep(masks=True))")
    ap.add_argument("--no-tf32", action="store_true")
    ap.add_argument("--check", action="store_true", help="dropout 0; compare both arms on the same seeded step")
    args = ap.parse_args()
    if args.vanilla and args.multi_frame:
        ap.error("--vanilla and --multi-frame are different models")
    if args.boxes is None:
        args.boxes = 60 if args.vanilla else 120
    if args.tracks is None:
        args.tracks = 50 if args.vanilla else 100
    from trackformer_b200.flat_adamw import reference_param_groups
    from trackformer_b200.model_factory import build_model, default_args, vanilla_args
    from trackformer_b200.train_step import TrainStep

    overrides = {"dropout": 0.0} if args.check else {}
    if args.masks:
        overrides["masks"] = True
    model_args = vanilla_args(tracking=True, dataset="mot", device="cuda:0", **overrides) if args.vanilla \
        else default_args(True, args.multi_frame, device="cuda:0", **overrides)
    if args.boxes > model_args.num_queries:
        ap.error(f"--boxes {args.boxes} exceeds the model's {model_args.num_queries} object queries")
    if not torch.cuda.is_available():
        sys.exit(f"track_train_bench needs a CUDA device (workload: {args.batch} x {args.height}x{args.width}, "
                 f"{model_args.num_queries} queries, {args.boxes} boxes, ~{args.tracks} track queries)")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = not args.no_tf32
    torch.manual_seed(0)
    model_a, criterion, _ = build_model(model_args)
    model_a.to(dev).train()
    criterion.to(dev).train()
    prepare = getattr(model_a.backbone[0], "prepare", None)
    if prepare is not None:
        prepare()                                       # the memory formats TrainStep gives the other arm's copy
    model_b = copy.deepcopy(model_a)
    g = torch.Generator().manual_seed(1)
    frames, targets = make_sample(g, dev, (args.height, args.width), args.boxes, args.batch, args.masks)
    seed = seed_for(args.tracks, args.boxes, model_a._track_query_false_positive_prob)

    # eager reference composition
    params_a = [p for p in model_a.parameters() if p.requires_grad]
    opt = torch.optim.AdamW(reference_param_groups(model_a), lr=2e-4, weight_decay=1e-4)
    wd = criterion.weight_dict

    def eager_step(tg, before_update=None):
        out, tg_out, _, _, _ = model_a(frames, tg)
        loss_dict = criterion(out, tg_out)
        loss = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        if before_update is not None:
            before_update()
        torch.nn.utils.clip_grad_norm_(params_a, 0.1)
        opt.step()
        return loss.detach()

    step = TrainStep(model_b, criterion, None, max_norm=0.1, use_graphs=True, example_frames=frames,
                     flat_adamw={"groups": reference_param_groups(model_b)}, track_bucket=args.bucket,
                     masks=args.masks)

    workload = ("vanilla DETR (100 object queries, softmax classifier, 21 classes)" if args.vanilla else
                "multi-frame model (500 queries, hidden 288, 8 levels)" if args.multi_frame else
                "300 object queries, 4 levels")
    if args.masks:
        workload += ", with the mask head"
    result = {"workload": "tracking train step, " + workload,
              "frame": [args.height, args.width], "batch": args.batch, "boxes": args.boxes, "track_bucket": args.bucket,
              "tf32": not args.no_tf32, "dropout": 0.0 if args.check else 0.1}

    if args.check:
        ta, tb = fresh(targets), fresh(targets)
        names_a = [n for n, p in model_a.named_parameters() if p.requires_grad]
        sample = {}

        def grab():
            flat = torch.cat([p.grad.reshape(-1) for p in params_a])
            idx = torch.randint(0, flat.numel(), (1 << 20,), generator=torch.Generator().manual_seed(7)).to(dev)
            sample["eager"] = flat[idx].clone()
            sample["idx"] = idx
        torch.manual_seed(seed)
        la = eager_step(ta, grab)
        torch.manual_seed(seed)
        lb = step(frames, tb)
        named_b = dict(model_b.named_parameters())
        flat_b = torch.cat([named_b[n].grad.reshape(-1) for n in names_a])
        gb = flat_b[sample["idx"]]
        ga = sample["eager"]
        same_idx = all(torch.equal(x[k], y[k]) for x, y in zip(ta, tb)
                       for k in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask"))
        rel = float((ga - gb).norm() / ga.norm().clamp_min(1e-30))
        cos = float((ga * gb).sum() / (ga.norm() * gb.norm()).clamp_min(1e-30))
        loss_rel = abs(float(la) - float(lb)) / max(abs(float(la)), 1e-12)
        ok = same_idx and loss_rel < 1e-3 and rel < 2e-2 and cos > 0.999
        differing = {k: int((x[k].long() != y[k].long()).sum()) if x[k].shape == y[k].shape else "shape"
                     for x, y in zip(ta, tb)
                     for k in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask")}
        result["check"] = {"ok": ok, "track_queries": len(ta[0]["track_query_boxes"]), "indices_equal": same_idx,
                           "differing_entries": differing,
                           "loss_eager": float(la), "loss_graphed": float(lb), "loss_rel_diff": loss_rel,
                           "grad_sample_rel_l2": rel, "grad_sample_cosine": cos}
        if not ok:
            print(json.dumps(result))
            sys.exit(1)

    def window(arm, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            torch.manual_seed(seed)
            tg = fresh(targets)
            if arm == "eager":
                eager_step(tg)
            else:
                step(frames, tg)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / max(n, 1), len(tg[0]["track_query_boxes"])

    window("eager", args.warmup)
    window("graphed", args.warmup)
    times = {"eager": [], "graphed": []}
    peak = {"eager": 0, "graphed": 0}
    for _ in range(args.rounds):
        for arm in ("eager", "graphed"):
            torch.cuda.reset_peak_memory_stats(dev)
            ms, k = window(arm, args.steps)
            times[arm].append(ms)
            peak[arm] = max(peak[arm], torch.cuda.max_memory_allocated(dev))
    med = {a: sorted(v)[len(v) // 2] for a, v in times.items()}
    name, limit = card()
    result.update({"track_queries": k, "ms_per_step_eager": med["eager"], "ms_per_step_graphed": med["graphed"],
                   "speedup": med["eager"] / med["graphed"], "windows_ms": times, "steps_per_window": args.steps,
                   "graph_captures": step.track_captures, "gpu": name, "power_limit": limit,
                   "peak_allocated_mib_eager": peak["eager"] / 2 ** 20,
                   "peak_allocated_mib_graphed": peak["graphed"] / 2 ** 20})
    print(json.dumps(result))


if __name__ == "__main__":
    main()
