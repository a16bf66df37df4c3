#!/usr/bin/env python
"""tools/gemm_bench.py -- the hand-written wgmma TF32 Linear (csrc/tf32_gemm.cu) against torch / cuBLAS.

Checks values (TF32 tolerance against an fp64 product) and times both with CUDA events (L2 flushed between
launches) on the long-token shapes of the C2 step.  Prints one JSON line per shape; --out writes the list.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [  # (M, K, N, what)
    (22223, 256, 256, "value_proj / output_proj"),
    (22223, 256, 384, "[sampling_offsets | attention_weights]"),
    (22223, 256, 1024, "FFN linear1"),
    (22223, 1024, 256, "FFN linear2"),
    (44446, 256, 256, "batch 2 value_proj"),
    (300, 256, 256, "decoder-sized"),
    (127, 32, 128, "tail smaller than one tile"),
]


def timed(fn, flush, iters):
    ts = []
    for _ in range(iters):
        flush.add_(1.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "gemm_bench.json"))
    args = ap.parse_args()
    from trackformer_b200 import ext
    m = ext.load()
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = True
    flush = torch.zeros(256 * 1024 * 1024 // 4, device=dev)
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    hbm = float(peaks.get("hbm_gbs", 3350.0))     # fallback: H100 SXM data sheet (3.35 TB/s HBM3), not measured
    out = []
    for (M, K, N, what) in SHAPES:
        g = torch.Generator(device="cpu").manual_seed(M + K + N)
        x = torch.randn(M, K, generator=g).to(dev)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        b = torch.randn(N, generator=g).to(dev)
        ref = (x.double() @ w.double().t() + b.double())
        for relu in (False, True):
            y = m.tf32_linear(x, w, b, relu)
            torch.cuda.synchronize()
            r = ref.clamp_min(0) if relu else ref
            err = float((y.double() - r).abs().max() / r.abs().max())
            assert err < 2e-3, (M, K, N, relu, err)
        y_lib = torch.nn.functional.linear(x, w, b)
        err_lib = float((y_lib.double() - ref).abs().max() / ref.abs().max())
        err_ours = float((m.tf32_linear(x, w, b, False).double() - ref).abs().max() / ref.abs().max())
        t_ours = timed(lambda: m.tf32_linear(x, w, b, False), flush, args.iters)
        t_lib = timed(lambda: torch.nn.functional.linear(x, w, b), flush, args.iters)
        # backward products of the same layer
        gy = torch.randn(M, N, generator=g).to(dev)
        rec_b = {}
        if m.tf32_linear_supported(M, N, K):
            dx_ref = gy.double() @ w.double()
            dw_ref = gy.double().t() @ x.double()
            dx = m.tf32_linear_dgrad(gy, w)
            dw = m.tf32_linear_wgrad(gy, x)
            torch.cuda.synchronize()
            e_dx = float((dx.double() - dx_ref).abs().max() / dx_ref.abs().max())
            e_dw = float((dw.double() - dw_ref).abs().max() / dw_ref.abs().max())
            assert e_dx < 2e-3 and e_dw < 2e-3, (M, K, N, e_dx, e_dw)
            rec_b = dict(dgrad_us=round(timed(lambda: m.tf32_linear_dgrad(gy, w), flush, args.iters), 2),
                         dgrad_cublas_us=round(timed(lambda: gy @ w, flush, args.iters), 2),
                         wgrad_us=round(timed(lambda: m.tf32_linear_wgrad(gy, x), flush, args.iters), 2),
                         wgrad_cublas_us=round(timed(lambda: gy.t() @ x, flush, args.iters), 2),
                         rel_err_dgrad=e_dx, rel_err_wgrad=e_dw)
        flops = 2.0 * M * N * K
        nbytes = 4.0 * (M * K + N * K + M * N)
        rec = dict(M=M, K=K, N=N, what=what, ours_us=round(t_ours, 2), cublas_us=round(t_lib, 2),
                   ours_tflops=round(flops / t_ours / 1e6, 1), cublas_tflops=round(flops / t_lib / 1e6, 1),
                   ours_gbs=round(nbytes / t_ours / 1e3, 1), hbm_frac=round(nbytes / t_ours / 1e3 / hbm, 3),
                   rel_err_ours=err_ours, rel_err_cublas_tf32=err_lib, **rec_b)
        out.append(rec)
        print(json.dumps(rec), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(out, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
