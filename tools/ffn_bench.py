#!/usr/bin/env python
"""tools/ffn_bench.py -- the encoder FFN (linear1 -> ReLU-dropout -> linear2, forward + backward) on the fused route
(fused_linear.ffn: activation and its gradient in the wgmma GEMM epilogues) against the composition it replaces
(fused_linear.linear + relu_dropout + fused_linear.linear), at the C2 token counts.

Both arms run in the same process and alternate round by round; each round times `--iters` forward + backward calls
with CUDA events.  Prints one JSON line per (rows, arm) with the median round, plus the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit not read"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[22223, 44446])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    from trackformer_b200 import deformable_transformer as dt
    from trackformer_b200 import fused_linear as fl
    torch.backends.cuda.matmul.allow_tf32 = True
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    layer = dt.DeformableTransformerEncoderLayer(256, 1024, 0.1).to(dev).train()
    info = card()
    for rows in args.rows:
        x = torch.randn(1, rows, 256, device=dev, requires_grad=True)
        gy = torch.randn(1, rows, 256, device=dev)
        assert fl.ffn_fusable(x, layer.linear1, layer.linear2, layer.dropout2)

        def fused():
            y = fl.ffn(x, layer.linear1, layer.linear2, layer.dropout2)
            y.backward(gy)

        def composed():
            a = fl.linear(x, layer.linear1.weight, layer.linear1.bias)
            h = fl.relu_dropout(a, layer.dropout2)
            y = fl.linear(h, layer.linear2.weight, layer.linear2.bias)
            y.backward(gy)

        arms = {"fused": fused, "composed": composed}
        times = {k: [] for k in arms}
        for fn in arms.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for name, fn in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    fn()
                b.record()
                b.synchronize()
                times[name].append(a.elapsed_time(b) * 1e3 / args.iters)
        for name, ts in times.items():
            ts.sort()
            print(json.dumps(dict(rows=rows, arm=name, fwd_bwd_us_median=round(ts[len(ts) // 2], 1),
                                  min_us=round(ts[0], 1), max_us=round(ts[-1], 1), card=info)), flush=True)


if __name__ == "__main__":
    main()
