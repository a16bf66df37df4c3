#!/usr/bin/env python
"""tools/ref_gpu_bench.py -- the REFERENCE's own model classes on the same GPU (test / measurement infrastructure).

Runs the unmodified reference Python package staged under the git-ignored baseline/_ref/ (oracle/stage_reference.py)
through its own training hot lines (src/trackformer/engine.py:126-151: model, SetCriterion with the scipy Hungarian
matcher, backward, clip_grad_norm_(0.1), AdamW), eagerly, as the reference runs, in two configurations:

  --msda ours     `import MultiScaleDeformableAttention` resolves to THIS repo's extension (trackformer_b200/ on sys.path):
                  the zero-edit drop-in route of INTEGRATION.md, executed on the GPU.  With --check the reference
                  model's outputs are compared with trackformer_b200's own model on the same weights and frame.
  --msda refcuda  the module is a thin shim over oracle/_ref/libmsda_refcuda.so, i.e. the reference's own CUDA kernels
                  compiled for sm_90a: "the reference on the same GPU" -- the honest GPU-vs-GPU denominator next to
                  the CPU arm of bench.py.

Prints one JSON line per run (frames/s of the C2 train step, 800x1333, batch 1, TF32 like bench.py).
"""
import argparse
import json
import os
import sys
import types

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGED = os.path.join(ROOT, "baseline", "_ref")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def import_reference(msda: str):
    vis = types.ModuleType("visdom")
    vis.Visdom = type("Visdom", (), {})
    sys.modules["visdom"] = vis
    if msda == "ours":
        sys.path.insert(0, os.path.join(ROOT, "trackformer_b200"))      # the extension under the reference's module name
        import MultiScaleDeformableAttention as M                       # noqa: F401
        assert "trackformer_b200" in M.__file__
    else:
        from oracle import refcuda
        assert refcuda.available(), "oracle/_ref/libmsda_refcuda.so missing (built only where /root/reference exists)"
        shim = types.ModuleType("MultiScaleDeformableAttention")
        shim.ms_deform_attn_forward = lambda v, s, l, a, step: refcuda.forward(v.contiguous(), s, l.contiguous(), a.contiguous())
        shim.ms_deform_attn_backward = lambda v, s, l, a, g, step: refcuda.backward(v.contiguous(), s, l.contiguous(),
                                                                                   a.contiguous(), g.contiguous())
        sys.modules["MultiScaleDeformableAttention"] = shim
    sys.path.insert(0, os.path.join(STAGED, "src"))
    import trackformer.models.backbone as bb
    bb.is_main_process = lambda: False                                  # never download weights
    from trackformer.models import build_model
    from trackformer.util.misc import nested_dict_to_namespace
    return build_model, nested_dict_to_namespace


def build_reference(build_model, to_ns, device, **overrides):
    def load(name):
        return yaml.safe_load(open(os.path.join(STAGED, "cfgs", name)))
    cfg = load("train.yaml")
    cfg.update(load("train_deformable.yaml"))
    cfg["device"] = str(device)
    cfg.update(overrides)
    torch.manual_seed(0)
    model, criterion, _ = build_model(to_ns(cfg))
    return model.to(device), criterion.to(device)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--msda", default="ours", choices=["ours", "refcuda"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", action="store_true", help="compare outputs with trackformer_b200's model (same weights)")
    ap.add_argument("--no-tf32", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert os.path.isdir(STAGED), "baseline/_ref is not staged (python oracle/stage_reference.py in the build container)"
    dev = torch.device("cuda:0")
    tf32 = not args.no_tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cudnn.benchmark = True
    import model_fixtures as mf
    build_model, to_ns = import_reference(args.msda)
    rec = {"msda": args.msda, "tf32": tf32}

    if args.check:
        from trackformer_b200.model_factory import build_model as ours_build, default_args
        ref_model, _ = build_reference(build_model, to_ns, dev)
        mf.canonical_weights_(ref_model, 0)
        ref_model.eval()
        torch.manual_seed(0)
        our_model, _, _ = ours_build(default_args(device=str(dev)))
        mf.canonical_weights_(our_model, 0)
        our_model.to(dev).eval()
        assert list(ref_model.state_dict()) == list(our_model.state_dict())
        frame = mf.make_images(1, [(800, 1333)], dev)[0][None]
        with torch.no_grad():
            a = ref_model(frame)[0]
            b = our_model(frame)[0]
        for k in ("pred_logits", "pred_boxes"):
            scale = float(a[k].abs().max())
            rec[f"max_rel_diff_{k}"] = float((a[k] - b[k]).abs().max()) / scale
        del ref_model, our_model
        torch.cuda.empty_cache()

    model, criterion = build_reference(build_model, to_ns, dev)
    model.train()
    criterion.train()
    params = [p for p in model.parameters() if p.requires_grad]
    opt = torch.optim.AdamW(mf.reference_optimizer_groups(model), lr=2e-4, weight_decay=1e-4)
    g = torch.Generator().manual_seed(1)
    frames = torch.randn(1, 3, 800, 1333, generator=g).to(dev)
    gt = torch.Generator().manual_seed(2)
    cxcy = torch.rand(20, 2, generator=gt) * 0.6 + 0.2
    wh = torch.rand(20, 2, generator=gt) * 0.25 + 0.05
    targets = [{"boxes": torch.cat([cxcy, wh], 1).to(dev), "labels": torch.zeros(20, dtype=torch.int64, device=dev)}]
    wd = criterion.weight_dict

    def step():
        outputs, tg, *_ = model(frames, targets)
        loss_dict = criterion(outputs, tg)
        losses = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
        opt.zero_grad()
        losses.backward()
        torch.nn.utils.clip_grad_norm_(params, 0.1)
        opt.step()
        return losses

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    rec.update({"metric": "frames/sec Deformable-DETR R50 800x1333 fwd+bwd (reference classes, eager)", "value": 1e3 / ms,
                "unit": "frames/s", "ms_per_step": ms, "steps": args.steps, "warmup": args.warmup,
                "loss": float(loss.detach()), "gpu": torch.cuda.get_device_name(0)})
    print(json.dumps(rec), flush=True)
    if args.out:
        json.dump(rec, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
