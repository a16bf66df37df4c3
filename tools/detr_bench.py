#!/usr/bin/env python
"""Vanilla DETR on one GPU: its attention kernels, its forward / training step with and without them, and MOTS
tracking latency.  Prints one JSON line with the card name and power limit (and writes it to --out when given).

--parts attn    Multi-head attention (hidden 256, 8 heads of 32 channels, batch --batch, second image padded on the right
                and bottom):
                  enc1050   encoder self-attention over the 25x42 stride-32 tokens of an 800x1333 frame
                  enc4200   the same with DC5 (50x84 tokens)
                  x100 / x137 / x300   decoder cross-attention from 100, 100 + 37 track and 300 queries onto 1050 tokens
                Arms (median of --repeats windows of --iters calls, CUDA events, TF32 Linears allowed):
                  core   the attention core alone (_DenseAttention), forward and forward + backward, dropout 0.1
                  ours   dense_attention.mha_forward (in-projection, core, out-projection)
                  stock  module(q, k, v, key_padding_mask) with need_weights=True (the reference's call) and False
                Forward-only arms in eval mode under no_grad, forward + backward in training mode.  Ours and stock are
                compared first (eval, TF32 off) and the largest difference is reported.
--parts model   DETR R50 (cfgs/train.yaml: 6 + 6 layers, 100 queries, random weights) on one 800x1333 frame, TF32:
                eval forward, an eager training step (forward + SetCriterion + backward, 20 boxes, dropout 0.1) and the
                graphed TrainStep (forward / backward CUDA graphs, loss in between, no optimizer) with the
                dense-attention kernels on (TFB200_DENSE_ATTN=1) and off (the stock nn.MultiheadAttention), alternated
                window by window in one process.  The eager arms are host-bound; the graphed one measures the GPU work.
                Then, dense attention on, where the softmax SetCriterion runs, alternated window by window:
                  one_graph   TrainStep(..., example_targets=...): forward, matching cost, device Hungarian matching,
                              fused loss and backward replayed from ONE graph
                  two_graph   forward / backward graphs with the device matching and the fused loss between them
                  host_match  the same two graphs with scipy on the host (criterion.device_matcher = False): one
                              device -> host copy of the cost per step
--parts mots    Per-frame latency of DETRSegmTracking (20-class head, masks) at 1080x1920 through GraphedDetector +
                DeviceTracker (host frame in, results out, device synchronised), --frames frames after --warmup.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {"enc1050": (None, (25, 42)), "enc4200": (None, (50, 84)), "x100": (100, (25, 42)), "x137": (137, (25, 42)),
         "x300": (300, (25, 42))}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:                                   # noqa: BLE001  (no nvidia-smi: the limit stays unknown)
        return torch.cuda.get_device_name(0), "unknown"


def time_ms(fn, iters, repeats):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return statistics.median(times)


def bench_attention(args, dev, result):
    from trackformer_b200 import dense_attention
    from trackformer_b200.dense_attention import _DenseAttention

    B = args.batch
    result["attn"] = {"batch": B, "iters": args.iters, "repeats": args.repeats, "cases": {}}
    for case in args.cases.split(","):
        lq, (h, w) = CASES[case]
        lk = h * w
        lq = lk if lq is None else lq
        g = torch.Generator().manual_seed(0)
        torch.manual_seed(0)
        mha = torch.nn.MultiheadAttention(256, 8, dropout=0.1).to(dev)
        tgt = torch.randn(lq, B, 256, generator=g).to(dev).requires_grad_(True)
        mem = torch.randn(lk, B, 256, generator=g).to(dev).requires_grad_(True)
        pad = torch.ones(B, h, w, dtype=torch.bool, device=dev)
        pad[0] = False
        pad[1:, : h * 4 // 5, : w * 3 // 4] = False
        pad = pad.flatten(1)
        query, key = (mem, mem) if lq == lk and case.startswith("enc") else (tgt, mem)
        gout = torch.randn(lq, B, 256, generator=g).to(dev)

        # agreement (eval, strict fp32)
        mha.eval()
        torch.backends.cuda.matmul.allow_tf32 = False
        with torch.no_grad():
            ours = dense_attention.mha_forward(mha, query, key, mem, pad)
            ref = mha(query, key, mem, key_padding_mask=pad, need_weights=False)[0]
        max_diff = float((ours - ref).abs().max())
        torch.backends.cuda.matmul.allow_tf32 = True

        e = 256
        with torch.no_grad():
            qh = torch.nn.functional.linear(query, mha.in_proj_weight[:e], mha.in_proj_bias[:e]).unflatten(-1, (8, 32))
            kh = torch.nn.functional.linear(key, mha.in_proj_weight[e:2 * e], mha.in_proj_bias[e:2 * e]).unflatten(-1, (8, 32))
            vh = torch.nn.functional.linear(mem, mha.in_proj_weight[2 * e:], mha.in_proj_bias[2 * e:]).unflatten(-1, (8, 32))
        qh, kh, vh = (t.contiguous().requires_grad_(True) for t in (qh, kh, vh))
        seed = torch.tensor([7], dtype=torch.int64, device=dev)
        gcore = gout.unflatten(-1, (8, 32))

        def core_fwd():
            with torch.no_grad():
                _DenseAttention.apply(qh, kh, vh, pad, None, 32 ** -0.5, 1.0)

        def core_fb():
            _DenseAttention.apply(qh, kh, vh, pad, seed, 32 ** -0.5, 0.9).backward(gcore)

        def ours_fwd():
            with torch.no_grad():
                dense_attention.mha_forward(mha, query, key, mem, pad)

        def ours_fb():
            dense_attention.mha_forward(mha, query, key, mem, pad).backward(gout)

        def stock(need_weights, backward):
            def fn():
                if backward:
                    mha(query, key, mem, key_padding_mask=pad, need_weights=need_weights)[0].backward(gout)
                else:
                    with torch.no_grad():
                        mha(query, key, mem, key_padding_mask=pad, need_weights=need_weights)
            return fn

        row = {"Lq": lq, "Lk": lk, "max_abs_diff_vs_stock_fp32": max_diff}
        mha.eval()
        row["core_fwd_ms"] = time_ms(core_fwd, args.iters, args.repeats)
        row["ours_fwd_ms"] = time_ms(ours_fwd, args.iters, args.repeats)
        row["stock_weights_fwd_ms"] = time_ms(stock(True, False), args.iters, args.repeats)
        row["stock_noweights_fwd_ms"] = time_ms(stock(False, False), args.iters, args.repeats)
        mha.train()
        row["core_fwd_bwd_ms"] = time_ms(core_fb, args.iters, args.repeats)
        row["ours_fwd_bwd_ms"] = time_ms(ours_fb, args.iters, args.repeats)
        row["stock_weights_fwd_bwd_ms"] = time_ms(stock(True, True), args.iters, args.repeats)
        row["stock_noweights_fwd_bwd_ms"] = time_ms(stock(False, True), args.iters, args.repeats)
        result["attn"]["cases"][case] = row
        print(case, json.dumps(row), flush=True)


def bench_model(args, dev, result):
    import copy
    from trackformer_b200 import dense_attention
    from trackformer_b200.train_step import TrainStep
    from trackformer_b200.model_factory import build_model, vanilla_args
    torch.manual_seed(0)
    model, criterion, _ = build_model(vanilla_args(device=str(dev)))
    model.to(dev)
    criterion.to(dev)
    g = torch.Generator().manual_seed(1)
    frame = torch.randn(1, 3, 800, 1333, generator=g).to(dev)
    boxes = torch.cat([torch.rand(20, 2, generator=g) * 0.6 + 0.2, torch.rand(20, 2, generator=g) * 0.2 + 0.05], 1)
    targets = [{"boxes": boxes.to(dev), "labels": torch.randint(0, 91, (20,), generator=g).to(dev)}]

    def forward():
        model.eval()
        with torch.no_grad():
            model(frame)

    def step():
        model.train()
        criterion.train()
        out, tg, _, _, _ = model(frame, targets)
        losses = criterion(out, tg)
        sum(losses[k] * criterion.weight_dict[k] for k in losses if k in criterion.weight_dict).backward()
        model.zero_grad(set_to_none=True)

    # the graphed training step (TrainStep: forward and backward replayed from CUDA graphs, loss in between): one
    # instance per arm, each captured with its own attention path on its own copy of the model
    graphed = {}
    for on in (True, False):
        dense_attention._ENABLED = on
        m = copy.deepcopy(model).train()
        graphed[on] = TrainStep(m, criterion, None, use_graphs=True, example_frames=frame)

    def graphed_step(on):
        return lambda: graphed[on](frame, targets)

    row = {}
    for name, fn, iters in (("forward", lambda on: forward, args.iters), ("train_step_eager", lambda on: step,
                            max(1, args.iters // 2)), ("train_step_graphed", graphed_step, args.iters)):
        times = {True: [], False: []}
        for rep in range(args.repeats):
            for on in (True, False):
                dense_attention._ENABLED = on
                times[on].append(time_ms(fn(on), iters, 1))
        dense_attention._ENABLED = True
        row[name + "_ms_dense_attn_on"] = statistics.median(times[True])
        row[name + "_ms_dense_attn_off"] = statistics.median(times[False])

    dense_attention._ENABLED = True
    host_criterion = copy.deepcopy(criterion)
    host_criterion.device_matcher = False
    arms = {"one_graph": TrainStep(copy.deepcopy(model).train(), criterion, None, use_graphs=True, example_frames=frame,
                                   example_targets=targets),
            "two_graph": graphed[True],
            "host_match": TrainStep(copy.deepcopy(model).train(), host_criterion, None, use_graphs=True,
                                    example_frames=frame)}
    assert arms["one_graph"].g_full is not None, "the detection step was not captured into one graph"
    times = {a: [] for a in arms}
    for rep in range(args.repeats):
        for a, st in arms.items():
            times[a].append(time_ms(lambda st=st: st(frame, targets), args.iters, 1))
    for a, v in times.items():
        row[f"train_step_{a}_ms"] = statistics.median(v)
    result["model"] = row
    print("model", json.dumps(row), flush=True)


def bench_mots(args, dev, result):
    import time
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.model_factory import build_model, vanilla_args
    from trackformer_b200.segmentation import PostProcessSegm
    torch.manual_seed(0)
    model, _, _ = build_model(vanilla_args(tracking=True, masks=True, dataset="mot", device=str(dev)))
    with torch.no_grad():
        model.class_embed.bias[0] += 6.0                # random weights: make class 0 confident so tracks exist
    model.to(dev).tracking()
    cfg = dict(public_detections=False, detection_obj_score_thresh=0.4, track_obj_score_thresh=0.4,
               detection_nms_thresh=0.9, track_nms_thresh=0.9, steps_termination=1, prev_frame_dist=1,
               inactive_patience=-1, reid_sim_threshold=0.0, reid_sim_only=False, reid_score_thresh=0.4,
               reid_greedy_matching=False)
    tracker = DeviceTracker(GraphedDetector(model), {"bbox": PostProcess(), "segm": PostProcessSegm()}, cfg, False)
    tracker.reset()
    g = torch.Generator().manual_seed(2)
    base = torch.randn(1, 3, 1080, 1920, generator=g)
    times = []
    with torch.no_grad():
        for i in range(args.warmup + args.frames):
            img = (base + 0.05 * torch.randn(1, 3, 1080, 1920, generator=g)).pin_memory()
            blob = {"img": img, "orig_size": torch.tensor([[1080, 1920]]), "size": torch.tensor([[1080, 1920]]),
                    "dets": torch.zeros(1, 0, 4)}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tracker.step(blob)
            torch.cuda.synchronize()
            if i >= args.warmup:
                times.append((time.perf_counter() - t0) * 1e3)
    row = {"frames": args.frames, "ms_per_frame_median": statistics.median(times), "ms_per_frame_min": min(times),
           "ms_per_frame_max": max(times), "tracks": len(tracker.get_results())}
    result["mots"] = row
    print("mots", json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="attn,model,mots")
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("detr_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    name, limit = card()
    result = {"gpu": name, "power_limit": limit}
    parts = args.parts.split(",")
    if "attn" in parts:
        bench_attention(args, dev, result)
    if "model" in parts:
        bench_model(args, dev, result)
    if "mots" in parts:
        bench_mots(args, dev, result)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
