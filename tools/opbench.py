#!/usr/bin/env python
"""Op-level micro-benchmark of the MSDeformAttn kernels (device pointers, CUDA-event timing).

  python tools/opbench.py [--cases c2_enc_model,c2_dec,...] [--variants 0,1,2] [--iters 30] [--once]

For every case it reports, per kernel variant, the median launch duration with the L2 flushed
between launches ("cold") and back-to-back ("warm"), the algorithmic bytes of the call
(SURVEY section 8: fwd 4*N*(S*M*D + 3*Lq*M*L*P + Lq*M*D), bwd 4*N*(2*S*M*D + 6*Lq*M*L*P + Lq*M*D))
and the achieved fraction of the measured HBM peak (MEASURED_PEAKS.json, else the 6.65 TB/s fallback).
``--once`` runs each kernel exactly once after one warm-up (for ncu).
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

C1 = [(60, 80), (30, 40), (15, 20), (8, 10)]
C2 = [(100, 167), (50, 84), (25, 42), (13, 21)]
C5 = [(135, 240), (68, 120), (34, 60), (17, 30)]

# name: (N, M, D, levels, P, Lq or None (= S, encoder), location distribution)
CASES = {
    "c2_enc_model": (1, 8, 32, C2, 4, None, "model"),
    "c2_enc_uniform": (1, 8, 32, C2, 4, None, "uniform"),
    # what bench.py's random-init model produces: sampling_offsets.weight = 0, bias = the 8-direction grid
    # (ms_deform_attn.py:34-42) -> every query samples the same pattern around its own reference point
    "c2_enc_init": (1, 8, 32, C2, 4, None, "model0"),
    "c2_enc_smooth": (1, 8, 32, C2, 4, None, "model0.1"),
    "c2_enc_init_n2": (2, 8, 32, C2, 4, None, "model0"),
    "c2_enc_model_n2": (2, 8, 32, C2, 4, None, "model"),
    "c2_dec": (1, 8, 32, C2, 4, 300, "boxes"),
    "c2_dec_n2": (2, 8, 32, C2, 4, 300, "boxes"),
    "c1_enc_model": (1, 8, 32, C1, 4, None, "model"),
    "c5_enc_model": (1, 8, 36, C5, 4, None, "model"),
    "c5_dec": (1, 8, 36, C5 * 2, 4, 800, "boxes"),
    # diagnostics: same number of queries / samples as c2_enc (22223 x 8 heads x 16), one level only
    "diag_l0_only": (1, 8, 32, [C2[0]], 16, 22223, "uniform"),
    "diag_l1_only": (1, 8, 32, [C2[1]], 16, 22223, "uniform"),
    "diag_l2_only": (1, 8, 32, [C2[2]], 16, 22223, "uniform"),
    "diag_l3_only": (1, 8, 32, [C2[3]], 16, 22223, "uniform"),
    "diag_l0_local": (1, 8, 32, [C2[0]], 16, 16700, "rowmajor"),
}

HEAD_DIRS = torch.tensor([[-1, -1], [-1, 0], [-1, 1], [0, -1], [0, 1], [1, -1], [1, 0], [1, 1]], dtype=torch.float32)


def make_case(name, dev, seed=0):
    N, M, D, hw, P, Lq, dist = CASES[name]
    g = torch.Generator().manual_seed(seed)
    shapes = torch.as_tensor(hw, dtype=torch.long)
    L = len(hw)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    enc = Lq is None
    Lq = S if enc else Lq
    value = torch.randn(N, S, M, D, generator=g)
    if dist == "uniform":
        loc = torch.rand(N, Lq, M, L, P, 2, generator=g)
    elif dist == "rowmajor":   # query q sits at pixel q of the (single) level, samples within +-3 px
        h, w = hw[0]
        q = torch.arange(Lq)
        cx = ((q % w).float() + 0.5) / w
        cy = ((q // w).float() + 0.5) / h
        ref = torch.stack([cx, cy], -1)[None, :, None, None, None, :]
        loc = ref + (torch.rand(N, Lq, M, L, P, 2, generator=g) - 0.5) * torch.tensor([6.0 / w, 6.0 / h])
    else:
        if enc:   # encoder reference points: pixel centres of every level (deformable_transformer.py:306-319)
            refs = []
            for (h, w) in hw:
                ys, xs = torch.meshgrid(torch.arange(h) + 0.5, torch.arange(w) + 0.5, indexing="ij")
                refs.append(torch.stack([xs.reshape(-1) / w, ys.reshape(-1) / h], -1))
            ref = torch.cat(refs, 0)[None, :, None, None, None, :].expand(N, S, 1, L, 1, 2)
            off = (HEAD_DIRS[torch.arange(M) % 8][None, None, :, None, None, :]
                   * torch.arange(1, P + 1, dtype=torch.float32)[None, None, None, None, :, None])
            jitter = float(dist[5:]) if len(dist) > 5 else 0.5
            off = off + jitter * torch.randn(N, Lq, M, L, P, 2, generator=g)       # "trained" per-sample jitter (pixels)
            # the reference normalises (x, y) offsets by (H, W) -- ops/modules/ms_deform_attn.py:78-79
            norm = shapes.to(torch.float32)[None, None, None, :, None, :]
            loc = ref + off / norm
        else:     # decoder: 4-d reference boxes (ms_deform_attn.py:80-82)
            cxcy = torch.rand(N, Lq, 1, 1, 1, 2, generator=g) * 0.8 + 0.1
            wh = torch.rand(N, Lq, 1, 1, 1, 2, generator=g) * 0.25 + 0.05
            off = (HEAD_DIRS[torch.arange(M) % 8][None, None, :, None, None, :]
                   * torch.arange(1, P + 1, dtype=torch.float32)[None, None, None, None, :, None])
            off = off + 0.5 * torch.randn(N, Lq, M, L, P, 2, generator=g)
            loc = cxcy + off / P * wh * 0.5
    attn = torch.softmax(torch.randn(N, Lq, M, L * P, generator=g), -1).view(N, Lq, M, L, P)
    gout = torch.randn(N, Lq, M * D, generator=g)
    t = [x.contiguous().to(dev) for x in (value, shapes, loc, attn, gout)]
    dims = dict(N=N, S=S, M=M, D=D, L=L, Lq=Lq, P=P)
    fwd_b = 4 * N * (S * M * D + 3 * Lq * M * L * P + Lq * M * D)
    bwd_b = 4 * N * (2 * S * M * D + 6 * Lq * M * L * P + Lq * M * D)
    return t, dims, fwd_b, bwd_b


def hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"]), "measured"
    return 6650.0, "fallback"


def time_kernel(fn, iters, flush, dev):
    times = []
    for _ in range(iters):
        if flush is not None:
            flush.add_(1.0)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e) * 1e3)
    times.sort()
    return times[len(times) // 2], times[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="c2_enc_model,c2_enc_uniform,c2_dec,c1_enc_model,c5_enc_model,c5_dec")
    ap.add_argument("--variants", default="0,1,2")
    ap.add_argument("--bwd-variants", default="0")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--once", action="store_true")
    ap.add_argument("--ref", action="store_true", help="also time the reference's own CUDA kernels (oracle/_ref)")
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "opbench.json"))
    args = ap.parse_args()

    from trackformer_b200 import ext
    msda = ext.load()
    dev = torch.device("cuda:0")
    peak, peak_src = hbm_peak()
    flush = torch.zeros(256 * 1024 * 1024 // 4, device=dev)       # 256 MB > 50 MB L2
    results = []
    for name in args.cases.split(","):
        (value, shapes, loc, attn, gout), dims, fwd_b, bwd_b = make_case(name, dev)
        for kind, variants, nbytes in (("fwd", args.variants, fwd_b), ("bwd", args.bwd_variants, bwd_b)):
            for v in [int(x) for x in variants.split(",")]:
                if kind == "fwd":
                    msda.set_variant(0 if v == -1 else (201 if v == -2 else v), 0)
                    if v in (-1, -2):      # TMA-staged tile kernel of the encoder (needs Lq == S); -2: four-warp variant
                        if dims["Lq"] != dims["S"]:
                            continue
                        flat_hw = [int(x) for x in shapes.cpu().flatten().tolist()]
                        fn = lambda: msda.ms_deform_attn_forward_enc_strict(value, shapes, loc, attn, flat_hw, 64)
                    else:
                        fn = lambda: msda.ms_deform_attn_forward(value, shapes, loc, attn, 64)
                else:
                    msda.set_variant(0, 0 if v == -1 else (203 if v == -3 else v))
                    if v in (-1, -3):      # TMA-staged backward tile kernel of the encoder (-3: coarse-level queries on the 8-lane-group kernel)
                        if dims["Lq"] != dims["S"]:
                            continue
                        flat_hw = [int(x) for x in shapes.cpu().flatten().tolist()]
                        fn = lambda: msda.ms_deform_attn_backward_enc_strict(value, shapes, loc, attn, gout, flat_hw, 64)
                    else:
                        fn = lambda: msda.ms_deform_attn_backward(value, shapes, loc, attn, gout, 64)
                fn()
                torch.cuda.synchronize()
                if args.once:
                    fn()
                    torch.cuda.synchronize()
                    continue
                for _ in range(3):
                    fn()
                cold, cold_min = time_kernel(fn, args.iters, flush, dev)
                warm, warm_min = time_kernel(fn, args.iters, None, dev)
                r = dict(case=name, kind=kind, variant=v, **dims, alg_bytes=nbytes,
                         cold_us=round(cold, 2), warm_us=round(warm, 2), cold_min_us=round(cold_min, 2),
                         cold_gbs=round(nbytes / cold / 1e3, 1), warm_gbs=round(nbytes / warm / 1e3, 1),
                         frac_cold=round(nbytes / cold / 1e3 / peak, 4), frac_warm=round(nbytes / warm / 1e3 / peak, 4),
                         peak_gbs=peak, peak_src=peak_src)
                results.append(r)
                print(json.dumps(r), flush=True)
    msda.set_variant(0, 0)
    # "the kernel to beat": the reference's own CUDA kernels compiled for sm_90a (oracle/_ref, test infrastructure)
    try:
        from oracle import refcuda
        have_ref = refcuda.available() and not args.once and args.ref
    except Exception:
        have_ref = False
    if have_ref:
        for name in args.cases.split(","):
            (value, shapes, loc, attn, gout), dims, fwd_b, bwd_b = make_case(name, dev)
            lib = refcuda._load()
            ws = torch.empty(lib.refcuda_ws_bytes(dims["N"], dims["M"], dims["D"], dims["L"], dims["Lq"], dims["P"], 4),
                             dtype=torch.uint8, device=dev)
            for kind, fn, nbytes in (("fwd", lambda: refcuda.forward(value, shapes, loc, attn, ws), fwd_b),
                                     ("bwd", lambda: refcuda.backward(value, shapes, loc, attn, gout, ws), bwd_b)):
                for _ in range(3):
                    fn()
                cold, _ = time_kernel(fn, max(5, args.iters // 3), flush, dev)
                warm, _ = time_kernel(fn, max(5, args.iters // 3), None, dev)
                r = dict(case=name, kind=kind, variant="reference_cuda", **dims, alg_bytes=nbytes, cold_us=round(cold, 2),
                         warm_us=round(warm, 2), cold_gbs=round(nbytes / cold / 1e3, 1), warm_gbs=round(nbytes / warm / 1e3, 1),
                         frac_cold=round(nbytes / cold / 1e3 / peak, 4), frac_warm=round(nbytes / warm / 1e3 / peak, 4),
                         peak_gbs=peak, peak_src=peak_src)
                results.append(r)
                print(json.dumps(r), flush=True)
            del ws
    if not args.once:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
