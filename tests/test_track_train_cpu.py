"""CPU tests of the tracking route of TrainStep and of the forced matching / row-masked loss it rests on.

The MSDeformAttn core has no CPU path, so these tests substitute the oracle's torch restatement for the CUDA function
(as tests/test_model_parity_cpu.py does); the route under test is product code.  On the CPU the decomposed tracking step
runs eagerly and takes the torch branch of ``SetCriterion.forward_stacked(..., track_queries=True)``: host forcing plus a
row mask -- the same decisions the device route makes with csrc/set_loss.cu."""
import copy
import ctypes
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import model_fixtures as mf
from test_model_parity_cpu import build, oracle_op  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = dict(enc_layers=1, dec_layers=2, num_queries=20, dropout=0.0)


def tracking_batch(seed, sizes=((96, 128),), n_boxes=7, prev_prev=False):
    """frames + targets with previous-frame images / targets, as in model_fixtures.run_train_step"""
    frames = torch.stack(mf.make_images(seed + 3, list(sizes)))
    targets = mf.make_targets(seed + 4, len(sizes), n_boxes, 1)
    prev_imgs = mf.make_images(seed + 5, list(sizes))
    for t, pim in zip(targets, prev_imgs):
        pt = {k: v.clone() for k, v in t.items()}
        pt["boxes"] = (pt["boxes"] + 0.01).clamp(0.05, 0.95)
        pt["track_ids"] = torch.cat([t["track_ids"][:-1], torch.tensor([99])])
        t["prev_target"] = pt
        t["prev_image"] = pim
        if prev_prev:
            ppt = {k: v.clone() for k, v in pt.items()}
            ppt["boxes"] = (ppt["boxes"] - 0.01).clamp(0.05, 0.95)
            t["prev_prev_target"] = ppt
            t["prev_prev_image"] = pim.flip(-1)
    return frames, targets


def reference_step(model, criterion, frames, targets):
    """the reference composition: model(samples, targets) + criterion + weighted sum + backward"""
    out, targets_out, _, _, _ = model(frames, targets)
    loss_dict = criterion(out, targets_out)
    wd = criterion.weight_dict
    total = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
    model.zero_grad(set_to_none=True)
    total.backward()
    return total.detach(), targets_out


def flat_of(step, model):
    """the reference model's gradients laid out like step.flat_grad"""
    flat = torch.zeros_like(step.flat_grad)
    named = dict(model.named_parameters())
    names = {id(p): n for n, p in step.model.named_parameters()}
    for p in step.params:
        o = (p.grad.data_ptr() - step.flat_grad.data_ptr()) // 4
        g = named[names[id(p)]].grad
        if g is not None:
            flat[o:o + p.numel()] = g.reshape(-1) if g.is_contiguous() else g.permute(0, 2, 3, 1).reshape(-1)
    return flat


def assert_same_bookkeeping(a, b):
    for ta, tb in zip(a, b):
        for key in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask"):
            assert torch.equal(ta[key], tb[key]), key
        assert torch.equal(ta["track_query_boxes"], tb["track_query_boxes"])


def make_step(model, criterion, bucket):
    from trackformer_b200.train_step import TrainStep
    return TrainStep(model, criterion, None, use_graphs=False, track_bucket=bucket)


@pytest.mark.parametrize("seed", [0, 3])
def test_decomposed_route_equals_the_eager_model_at_bucket_1(oracle_op, seed):
    model, criterion = build(True, False, **SMALL)
    mf.canonical_weights_(model, seed)
    model.train()
    ref = copy.deepcopy(model)
    frames, targets = tracking_batch(seed, sizes=((96, 128), (96, 128)))
    ref_targets = copy.deepcopy(targets)
    step = make_step(model, criterion, 1)
    assert step._tracking_route(targets) == "track"

    torch.manual_seed(1234)
    loss = step(frames, targets)
    after_step = torch.rand(4)
    torch.manual_seed(1234)
    ref_loss, ref_targets = reference_step(ref, criterion, frames, ref_targets)
    after_ref = torch.rand(4)

    assert torch.equal(after_step, after_ref)                     # the CPU generator was consumed identically
    assert_same_bookkeeping(targets, ref_targets)
    assert len(targets[0]["track_query_boxes"]) > 0
    torch.testing.assert_close(loss, ref_loss, rtol=1e-5, atol=1e-6)
    ref_flat = flat_of(step, ref)
    torch.testing.assert_close(step.flat_grad, ref_flat, rtol=2e-4, atol=1e-6 * float(ref_flat.abs().max()))


@pytest.mark.parametrize("bucket", [4, 16])
def test_filler_rows_change_nothing(oracle_op, bucket):
    model, criterion = build(True, False, **SMALL)
    mf.canonical_weights_(model, 1)
    model.train()
    other = copy.deepcopy(model)
    frames, targets = tracking_batch(1)
    targets_b = copy.deepcopy(targets)
    plain, padded = make_step(other, criterion, 1), make_step(model, criterion, bucket)
    torch.manual_seed(7)
    la = plain(frames, targets_b)
    torch.manual_seed(7)
    lb = padded(frames, targets)
    assert_same_bookkeeping(targets, targets_b)
    k = len(targets[0]["track_query_boxes"])
    assert k % bucket != 0                                        # fillers present
    torch.testing.assert_close(lb, la, rtol=1e-5, atol=1e-6)
    scale = float(plain.flat_grad.abs().max())
    torch.testing.assert_close(padded.flat_grad, plain.flat_grad, rtol=2e-4, atol=2e-6 * scale)


def random_tracking_targets(g, n_boxes, n_track, n_fp, nq):
    """targets as add_track_queries_to_targets leaves them: n_track track rows (the last n_fp false positives)
    followed by nq object rows"""
    t = {"boxes": torch.cat([torch.rand(n_boxes, 2, generator=g) * 0.6 + 0.2,
                             torch.rand(n_boxes, 2, generator=g) * 0.2 + 0.05], 1),
         "labels": torch.zeros(n_boxes, dtype=torch.int64)}
    is_track = torch.zeros(n_track + nq, dtype=torch.bool)
    is_track[:n_track] = True
    fp = torch.zeros_like(is_track)
    fp[n_track - n_fp:n_track] = True
    t["track_queries_mask"], t["track_queries_fal_pos_mask"] = is_track, fp
    t["track_query_match_ids"] = torch.randperm(n_boxes, generator=g)[:n_track - n_fp]
    t["track_query_boxes"] = torch.rand(n_track, 4, generator=g)
    return t


def pad_rows(x, n_track, kb, dim):
    """insert kb - n_track filler rows after the track rows of dimension ``dim``"""
    shape = (*x.shape[:dim], kb - n_track, *x.shape[dim + 1:])
    fill = torch.rand(shape) if x.shape[-1] == 4 else torch.randn(shape) * 3         # boxes stay valid cxcywh
    return torch.cat([x.narrow(dim, 0, n_track), fill, x.narrow(dim, n_track, x.shape[dim] - n_track)], dim)


def test_host_forced_matching_with_fillers_equals_forward():
    from trackformer_b200.matcher import HungarianMatcher
    m = HungarianMatcher(2.0, 5.0, 2.0, focal_loss=True)
    g = torch.Generator().manual_seed(0)
    nq, n_track, kb, n_layers = 12, 5, 8, 3
    targets = [random_tracking_targets(g, 6, n_track, 1, nq), random_tracking_targets(g, 9, n_track, 2, nq)]
    logits = torch.randn(n_layers, 2, n_track + nq, 20, generator=g)
    boxes = torch.rand(n_layers, 2, n_track + nq, 4, generator=g)
    want = [m.forward({"pred_logits": logits[i], "pred_boxes": boxes[i]}, targets) for i in range(n_layers)]
    padded_targets = [dict(t, track_query_padding=torch.arange(kb) >= n_track) for t in targets]
    got = m.match_layers_forced(pad_rows(logits, n_track, kb, 2), pad_rows(boxes, n_track, kb, 2), padded_targets)
    for layer_want, layer_got in zip(want, got):
        for (ws, wt), (gs, gt) in zip(layer_want, layer_got):
            back = torch.where(gs >= kb, gs - (kb - n_track), gs)
            assert not ((gs >= n_track) & (gs < kb)).any()        # no filler row is ever matched
            assert torch.equal(back, ws) and torch.equal(gt, wt)
    # without fillers the host route is forward itself
    got = m.match_layers_forced(logits, boxes, targets)
    for layer_want, layer_got in zip(want, got):
        for (ws, wt), (gs, gt) in zip(layer_want, layer_got):
            assert torch.equal(gs, ws) and torch.equal(gt, wt)


def test_masked_torch_loss_equals_unpadded_and_fillers_get_no_gradient():
    from trackformer_b200.model_factory import build_model, default_args
    _, criterion, _ = build_model(default_args(True, False, device="cpu", **SMALL))
    g = torch.Generator().manual_seed(1)
    nq, n_track, kb, n_layers = 20, 3, 8, 2
    targets = [random_tracking_targets(g, 5, n_track, 1, nq)]
    logits = torch.randn(n_layers, 1, n_track + nq, 20, generator=g)
    boxes = torch.rand(n_layers, 1, n_track + nq, 4, generator=g)
    ref = criterion(dict(pred_logits=logits[-1], pred_boxes=boxes[-1],
                         aux_outputs=[{"pred_logits": logits[0], "pred_boxes": boxes[0]}]), targets)
    pl = pad_rows(logits, n_track, kb, 2).requires_grad_(True)
    pb = pad_rows(boxes, n_track, kb, 2).requires_grad_(True)
    padded_targets = [dict(t, track_query_padding=torch.arange(kb) >= n_track) for t in targets]
    got = criterion.forward_stacked(pl, pb, padded_targets, track_queries=True)
    assert set(got) == set(ref)
    for k in ref:
        torch.testing.assert_close(got[k], ref[k], rtol=1e-5, atol=1e-6, msg=k)
    wd = criterion.weight_dict
    gl, gb = torch.autograd.grad(sum(got[k] * wd[k] for k in got if k in wd), (pl, pb))
    assert float(gl[:, :, n_track:kb].abs().max()) == 0.0 and float(gb[:, :, n_track:kb].abs().max()) == 0.0
    assert float(gl[:, :, :n_track].abs().max()) > 0.0
    # without the keyword, routing is as before: tracking targets take forward()
    plain = criterion.forward_stacked(logits, boxes, targets)
    for k in ref:
        torch.testing.assert_close(plain[k], ref[k], rtol=0, atol=0, msg=k)


@pytest.mark.parametrize("case", ["prev_prev", "backprop_prev_frame", "no_prev_image"])
def test_fallback_routes_equal_model_plus_criterion(oracle_op, case):
    overrides = dict(SMALL, track_backprop_prev_frame=(case == "backprop_prev_frame"))
    model, criterion = build(True, False, **overrides)
    mf.canonical_weights_(model, 2)
    model.train()
    ref = copy.deepcopy(model)
    frames, targets = tracking_batch(2, prev_prev=(case == "prev_prev"))
    if case == "no_prev_image":
        targets = [{k: v for k, v in t.items() if not k.startswith("prev")} for t in targets]
    ref_targets = copy.deepcopy(targets)
    step = make_step(model, criterion, 4)
    assert step._tracking_route(targets) == ("detect" if case == "no_prev_image" else "eager")
    torch.manual_seed(5)
    loss = step(frames, targets)
    torch.manual_seed(5)
    if case == "no_prev_image":                      # the detection step of a tracking model: no track queries
        out = ref(frames)[0]
        loss_dict = criterion(out, ref_targets)
        ref_loss = sum(loss_dict[k] * criterion.weight_dict[k] for k in loss_dict if k in criterion.weight_dict)
        ref.zero_grad(set_to_none=True)
        ref_loss.backward()
    else:
        ref_loss, ref_targets = reference_step(ref, criterion, frames, ref_targets)
        assert_same_bookkeeping(targets, ref_targets)
    torch.testing.assert_close(loss, ref_loss.detach(), rtol=1e-5, atol=1e-6)
    ref_flat = flat_of(step, ref)
    torch.testing.assert_close(step.flat_grad, ref_flat, rtol=2e-4, atol=1e-6 * float(ref_flat.abs().max()))


def test_mask_models_stay_rejected():
    from trackformer_b200.model_factory import build_model, default_args
    from trackformer_b200.train_step import TrainStep
    model, criterion, _ = build_model(default_args(True, False, device="cpu", masks=True, **SMALL))
    with pytest.raises(NotImplementedError):
        TrainStep(model, criterion, None, use_graphs=False, track_bucket=4)


# ---- data parallel: ranks with different buckets -------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import trackformer_b200.msda_module as mm
    from oracle.torch_ref import msda_core_torch

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    mm.MSDeformAttnFunction = _OracleFn
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        model, criterion = build(True, False, **SMALL)
        mf.canonical_weights_(model, 0)
        model.train()
        step = make_step(model, criterion, 3 if rank == 0 else 8)
        losses = []
        for i in range(2):
            frames, targets = tracking_batch(10 * i + rank, n_boxes=5 + rank)
            if rank == 1 and i == 1:                  # one rank on the eager fallback route in the same step
                targets[0]["prev_prev_image"] = targets[0]["prev_image"].flip(-1)
                targets[0]["prev_prev_target"] = {k: v.clone() for k, v in targets[0]["prev_target"].items()}
            torch.manual_seed(100 + 10 * i + rank)
            losses.append(float(step(frames, targets)))
        torch.save({"grad": step.flat_grad.clone(), "k": len(targets[0]["track_query_boxes"])},
                   os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_ranks_on_different_buckets_end_with_equal_gradients(tmp_path):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    got = [torch.load(tmp_path / f"rank{r}.pt") for r in range(world)]
    assert torch.equal(got[0]["grad"], got[1]["grad"])
    assert float(got[0]["grad"].abs().sum()) > 0


# ---- C entry points ------------------------------------------------------------------------------------------------
def test_new_entry_points_reject_bad_arguments():
    from trackformer_b200 import _build, ext
    lib = ctypes.CDLL(_build.build_library())
    vp, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    cost = lib.tfb200_match_cost_track_f32
    cost.restype = i
    cost.argtypes = [vp] * 6 + [i] * 5 + [f] * 5 + [vp]
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, vp)
    assert cost(None, p, p, p, p, p, 1, 1, 4, 20, 3, 1, 1, 1, .25, 2, None) == -1       # NULL logits
    assert cost(p, p, p, p, None, p, 1, 1, 4, 20, 3, 1, 1, 1, .25, 2, None) == -1       # NULL row_pin
    assert cost(p, p, p, p, p, p, 1, 0, 4, 20, 3, 1, 1, 1, .25, 2, None) == -2          # B = 0
    assert cost(p, p, p, p, p, p, 1, 1, 4, 20, 0, 1, 1, 1, .25, 2, None) == -2          # T = 0
    assert cost(p, p, p, p, p, p, 1, 1, 4, 20, 1 << 20, 1, 1, 1, .25, 2, None) == -2    # T beyond shared memory
    assert cost(p, p, p, p, p, p, 0, 1, 4, 20, 3, 1, 1, 1, .25, 2, None) == 0           # no layers: no-op
    loss = lib.tfb200_set_loss_fwd_masked_f32
    loss.restype = i
    loss.argtypes = [vp] * 18 + [i] * 5 + [f] * 2 + [vp]
    args = [p] * 18
    no_mask = list(args)
    no_mask[9] = None
    assert loss(*no_mask, 1, 1, 4, 20, 3, .25, 2, None) == -1                           # NULL row_valid
    no_logits = list(args)
    no_logits[0] = None
    assert loss(*no_logits, 1, 1, 4, 20, 3, .25, 2, None) == -1
    assert loss(*args, 0, 1, 4, 20, 3, .25, 2, None) == -2                              # K = 0
    assert loss(*args, 1, 1, 4, 20, 0, .25, 2, None) == -2                              # T = 0
    m = ext.load()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.match_cost_track(torch.zeros(1, 1, 4, 20), torch.zeros(1, 1, 4, 4), torch.zeros(3, dtype=torch.int64),
                           torch.zeros(3, 4), torch.zeros(4, dtype=torch.int32), 1.0, 1.0, 1.0, 0.25, 2.0)
    with pytest.raises(RuntimeError, match="dtypes"):
        m.set_loss_forward_masked(torch.zeros(1, 1, 4, 20), torch.zeros(1, 1, 4, 4), torch.zeros(1, 3, dtype=torch.int64),
                                  torch.zeros(1, 3, dtype=torch.int64), torch.zeros(3, dtype=torch.int64),
                                  torch.zeros(3, 4), torch.zeros(2, dtype=torch.int32), torch.zeros(1), torch.ones(1),
                                  torch.ones(4, dtype=torch.uint8), 0.25, 2.0)
