"""GPU tests of the softmax (vanilla-DETR) set criterion on the device (csrc/set_loss.cu, SoftmaxCls) and of the
TrainStep routes it opens: the one-graph detection step and the graphed tracking step.  Strict fp32 throughout.

  * matching cost (match_cost_softmax, match_cost_track_softmax), plain and forced, with and without filler rows, against
    an fp64 torch restatement of models/matcher.py; the device solver on the kernel's cost against scipy;
  * loss values and gradients of the fused route of forward_stacked against its fp64 torch restatement and against
    the reference's own SetCriterion (tests/golden/softmax_criterion.npz);
  * TrainStep: vanilla detection captured into one graph, with the host solver disabled, against the uncaptured step
    and the detr_train_step_det fixture; the graphed vanilla tracking step against the eager composition and the
    detr_train_step_tracking fixture."""
import copy

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

import detr_fixtures as df
import model_fixtures as mf
import softmax_criterion_fixtures as smf
from conftest import load_golden

pytestmark = pytest.mark.gpu

SMALL = dict(enc_layers=1, dec_layers=2, num_queries=20, dropout=0.0)
# of the cost matrix's scale: the GIoU term of a tiny pair (shared with the focal cost) carries the fp32 rounding of its
# corners, ~1e-5 of the scale at C + 1 = 21
COST_TOL = 2e-5
# tiny boxes (w, h ~ 1e-3): their corners cx -+ w/2 carry fp32 rounding of ~3e-5 of the width and the GIoU gradient scales
# with 1 / width, so the rows predicting them are checked on their own scale at this tolerance
GRAD_TINY_TOL = 3e-4


def close_boxes(got, want, boxes):
    """box gradients: tiny predicted boxes on their own scale at GRAD_TINY_TOL, every other row at 1e-4"""
    tiny = (boxes[..., 2:] < 2e-3).any(-1)
    for rows, rtol in ((~tiny, 1e-4), (tiny, GRAD_TINY_TOL)):
        if bool(rows.any()):
            w = want[rows]
            torch.testing.assert_close(got[rows], w, rtol=rtol, atol=2e-6 * float(w.abs().max()) if rtol < 2e-4
                                       else rtol * float(w.abs().max()))


@pytest.fixture()
def strict_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.fixture(scope="module")
def gold():
    return load_golden("softmax_criterion", "")


def criterion_for(case, fp="fp1"):
    from trackformer_b200.criterion import SetCriterion
    from trackformer_b200.matcher import HungarianMatcher
    matcher = HungarianMatcher(smf.COST_CLASS, smf.COST_BBOX, smf.COST_GIOU, focal_loss=False)
    return SetCriterion(case["C"] - 1, matcher, {}, smf.EOS_COEF, ["labels", "boxes", "cardinality"], False, 0.25, 2.0,
                        True, smf.FP_WEIGHT[fp])


def weighted_total(losses, w):
    names = ("loss_ce", "loss_bbox", "loss_giou")
    return sum(float(w[i, k]) * losses[n if k == smf.K - 1 else f"{n}_{k}"] for i, n in enumerate(names)
               for k in range(smf.K))


def padded(case, extra):
    """logits / boxes with ``extra`` filler rows after the track rows, and the targets that mark them"""
    n = case["n_track"]
    g = torch.Generator().manual_seed(extra)
    lg, bx = case["logits"], case["boxes"]
    fl = torch.randn(*lg.shape[:2], extra, lg.shape[3], generator=g) * 3
    fb = torch.rand(*bx.shape[:2], extra, 4, generator=g) * 0.4 + 0.1
    lg = torch.cat([lg[:, :, :n], fl, lg[:, :, n:]], 2).contiguous()
    bx = torch.cat([bx[:, :, :n], fb, bx[:, :, n:]], 2).contiguous()
    targets = [dict(t, track_query_padding=torch.arange(n + extra) >= n) for t in case["targets"]]
    return lg, bx, targets


def to(targets, dev, dtype=torch.float32):
    return [{k: (v.to(dev, dtype) if k == "boxes" else v.to(dev)) for k, v in t.items()} for t in targets]


# ---- matching cost ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fillers", [0, 5])
@pytest.mark.parametrize("name", list(smf.CASES))
def test_cost_against_fp64(cuda_device, strict_fp32, name, fillers):
    from trackformer_b200 import ext
    from trackformer_b200.matcher import HungarianMatcher
    case = smf.make_case(name)
    lg, bx, targets = padded(case, fillers) if fillers else (case["logits"], case["boxes"], case["targets"])
    m = HungarianMatcher(smf.COST_CLASS, smf.COST_BBOX, smf.COST_GIOU, focal_loss=False)
    k, bs, nq, _ = lg.shape
    tgt_ids = torch.cat([t["labels"] for t in targets])
    tgt_boxes = torch.cat([t["boxes"] for t in targets])
    ref = m._cost(lg.double().flatten(0, 2), bx.double().flatten(0, 2), tgt_ids, tgt_boxes.double()).view(k, bs, nq, -1)
    pin = m.row_pin(targets, nq, "cpu")
    ref_forced = m.force_cost(ref, pin)
    dev = cuda_device
    plain = ext.load().match_cost_softmax(lg.to(dev), bx.to(dev), tgt_ids.to(dev), tgt_boxes.to(dev), smf.COST_CLASS,
                                          smf.COST_BBOX, smf.COST_GIOU).view(k, bs, nq, -1).cpu().double()
    forced = ext.load().match_cost_track_softmax(lg.to(dev), bx.to(dev), tgt_ids.to(dev), tgt_boxes.to(dev),
                                                 pin.to(dev), smf.COST_CLASS, smf.COST_BBOX, smf.COST_GIOU).cpu().double()
    for got, want in ((plain, ref), (forced, ref_forced)):
        assert torch.equal(torch.isinf(got), torch.isinf(want))
        fin = torch.isfinite(want)
        err = float((got[fin] - want[fin]).abs().max() / want[fin].abs().max())
        assert err <= COST_TOL, f"cost vs fp64: {err:.3e}"
    free = torch.isfinite(ref_forced) & (ref_forced != -1)
    assert torch.equal(forced[free], plain[free])                  # the same entries bit for bit

    # the device solver on the kernel's forced cost picks scipy's pairs on that same cost
    sizes = [len(t["boxes"]) for t in targets]
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32, device=dev)
    src, tgt, status = ext.load().lsa(forced.float().to(dev), off, max(sizes))
    assert int(status[0]) == 0
    src, tgt = src.cpu(), tgt.cpu()
    c32 = forced.float()
    for layer in range(k):
        for b in range(bs):
            r, c = linear_sum_assignment(c32[layer, b, :, off[b]:off[b + 1]].numpy())
            assert np.array_equal(src[layer, off[b]:off[b + 1]].numpy(), r)
            assert np.array_equal(tgt[layer, off[b]:off[b + 1]].numpy() - int(off[b]), c)


# ---- loss ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fillers", [0, 7])
@pytest.mark.parametrize("fp", list(smf.FP_WEIGHT))
@pytest.mark.parametrize("name", list(smf.CASES))
def test_fused_loss_against_fp64_and_reference(cuda_device, strict_fp32, gold, monkeypatch, name, fp, fillers):
    from trackformer_b200 import criterion as crit_mod
    from trackformer_b200.matcher import HungarianMatcher
    case = smf.make_case(name)
    lg, bx, targets = padded(case, fillers) if fillers else (case["logits"], case["boxes"], case["targets"])
    crit = criterion_for(case, fp)

    # fp64 torch restatement (host matching, CPU)
    l64 = lg.double().requires_grad_(True)
    b64 = bx.double().requires_grad_(True)
    ref = crit.double().forward_stacked(l64, b64, to(targets, "cpu", torch.float64), track_queries=True)
    rl, rb = torch.autograd.grad(weighted_total(ref, case["weights"]), (l64, b64))

    # fused route: no host solver, one autograd Function
    calls = []
    real = crit_mod._SetLossSoftmax.apply
    monkeypatch.setattr(crit_mod._SetLossSoftmax, "apply", lambda *a: calls.append(1) or real(*a))
    monkeypatch.setattr(HungarianMatcher, "_assign", staticmethod(lambda *a: pytest.fail("host solver reached")))
    crit = crit.float().to(cuda_device)
    l32 = lg.to(cuda_device).requires_grad_(True)
    b32 = bx.to(cuda_device).requires_grad_(True)
    got = crit.forward_stacked(l32, b32, to(targets, cuda_device), track_queries=True)
    gl, gb = torch.autograd.grad(weighted_total(got, case["weights"]), (l32, b32))
    assert calls == [1]

    assert set(got) == set(ref)
    for key in ref:
        g, r = float(got[key]), float(ref[key])
        if key.startswith(("cardinality_error", "class_error")):
            assert g == pytest.approx(r, abs=1e-4), key                  # counts: exact up to the fp32 division
        else:
            assert g == pytest.approx(r, rel=2e-5, abs=1e-7), key
    scale_l = float(rl.abs().max())
    torch.testing.assert_close(gl.cpu().double(), rl, rtol=1e-4, atol=2e-6 * scale_l)
    close_boxes(gb.cpu().double(), rb, bx)
    if fillers:
        n = case["n_track"]
        assert float(gl[:, :, n:n + fillers].abs().max()) == 0.0 and float(gb[:, :, n:n + fillers].abs().max()) == 0.0
        return

    # the reference's own SetCriterion
    pre = f"{name}_{fp}_"
    for base in ("loss_ce", "loss_bbox", "loss_giou", "cardinality_error"):
        vals = np.array([float(got[base if k == smf.K - 1 else f"{base}_{k}"]) for k in range(smf.K)])
        np.testing.assert_allclose(vals, gold[pre + base], rtol=2e-5, atol=1e-4 if base == "cardinality_error" else 1e-7,
                                   err_msg=base)
    np.testing.assert_allclose(float(got["class_error"]), gold[pre + "class_error"], atol=1e-3)
    rows = gold[pre + "grad_logits_rows"]
    g_rows = gold[pre + "grad_logits"]
    np.testing.assert_allclose(gl.cpu().numpy()[rows], g_rows, rtol=1e-4, atol=2e-6 * float(np.abs(g_rows).max()))
    g_boxes = gold[pre + "grad_boxes"]
    close_boxes(gb.cpu().double(), torch.from_numpy(g_boxes).double(), bx)


# ---- detection step in one graph ---------------------------------------------------------------------------------------
def det_batch(seed, n_boxes, dev, sizes=((160, 224), (160, 224))):
    frames = torch.stack(mf.make_images(seed + 3, list(sizes), dev))
    targets = mf.make_targets(seed + 4, len(sizes), n_boxes, 1, dev)
    return frames, [{"boxes": t["boxes"], "labels": t["labels"]} for t in targets]


def test_vanilla_detection_step_runs_in_one_graph(cuda_device, strict_fp32, monkeypatch):
    from trackformer_b200.matcher import HungarianMatcher
    from trackformer_b200.train_step import TrainStep
    monkeypatch.setattr(HungarianMatcher, "_assign", staticmethod(lambda *a: pytest.fail("host solver reached")))
    model, criterion = df.build(False, False, device=str(cuda_device), **SMALL)
    mf.canonical_weights_(model, 0)
    model.to(cuda_device).train()
    criterion.to(cuda_device)
    plain_model = copy.deepcopy(model)
    frames, example = det_batch(0, 6, cuda_device)
    step = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames, example_targets=example)
    assert step.g_full is not None
    plain = TrainStep(plain_model, criterion, None, use_graphs=False)
    replays = []
    real_replay = step.g_full.replay
    step.g_full.replay = lambda: replays.append(1) or real_replay()
    for i, n in enumerate((6, 6, 4, 6, 9)):
        frames_i, targets = det_batch(10 + i, n, cuda_device)
        loss = step(frames_i, targets)
        want = plain(frames_i, targets)
        torch.testing.assert_close(loss, want, rtol=1e-5, atol=1e-6)
        scale = float(plain.flat_grad.abs().max())
        torch.testing.assert_close(step.flat_grad, plain.flat_grad, rtol=1e-4, atol=1e-6 * scale)
    assert len(replays) == 3                                       # the steps with the captured box counts


def test_one_graph_step_reproduces_detr_train_step_det(cuda_device, strict_fp32):
    from trackformer_b200.train_step import TrainStep
    gold = load_golden("train_step_det", "detr_")
    model, criterion = df.build(False, False, device=str(cuda_device), dropout=0.0)
    mf.canonical_weights_(model, 0)
    model.to(cuda_device).train()
    criterion.to(cuda_device).train()
    sizes = [(160, 224), (160, 224)]
    frames = torch.stack(mf.make_images(3, sizes, cuda_device))
    targets = mf.make_targets(4, len(sizes), 6, 1, cuda_device)
    step = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames, example_targets=targets)
    assert step.g_full is not None
    loss = step(frames, targets)
    named = dict(model.named_parameters())
    res = {"loss_total": loss.cpu().numpy()}
    for key in mf.GRAD_KEYS:
        if key in named:
            res["grad/" + key] = named[key].grad.cpu().numpy()
    res["grad_global_norm"] = np.array(float(step.flat_grad.double().norm()))
    sub = {k: v for k, v in gold.items() if k in res}
    assert "loss_total" in sub and "grad_global_norm" in sub
    df.check(res, sub, rtol=5e-3, rel_atol=2e-3)


# ---- graphed tracking step -----------------------------------------------------------------------------------------------
def track_batch(seed, dev, sizes=((128, 160),), n_boxes=7):
    frames = torch.stack(mf.make_images(seed + 3, list(sizes), dev))
    targets = mf.make_targets(seed + 4, len(sizes), n_boxes, 1, dev)
    for t, pim in zip(targets, mf.make_images(seed + 5, list(sizes), dev)):
        pt = {k: v.clone() for k, v in t.items()}
        pt["boxes"] = (pt["boxes"] + 0.01).clamp(0.05, 0.95)
        pt["track_ids"] = torch.cat([t["track_ids"][:-1], torch.tensor([99]).to(dev)])
        t["prev_target"], t["prev_image"] = pt, pim
    return frames, targets


def test_graphed_tracking_step_reproduces_detr_train_step_tracking(cuda_device, strict_fp32):
    from trackformer_b200.train_step import TrainStep
    gold = load_golden("train_step_tracking", "detr_")
    model, criterion = df.build(True, False, device=str(cuda_device), dropout=0.0)
    mf.canonical_weights_(model, 0)
    model.to(cuda_device).train()
    criterion.to(cuda_device).train()
    frames, targets = track_batch(0, cuda_device)
    step = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames, track_bucket=4)
    assert step._tracking_route(targets) == "track"
    torch.manual_seed(1234)
    loss = step(frames, targets)
    named = dict(model.named_parameters())
    res = {"loss_total": loss.cpu().numpy(), "grad_global_norm": np.array(float(step.flat_grad.double().norm()))}
    for key in mf.GRAD_KEYS:
        if key in named:
            res["grad/" + key] = named[key].grad.cpu().numpy()
    for i, t in enumerate(targets):
        for key in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask"):
            res[f"idx/{i}/{key}"] = t[key].long().cpu().numpy()
        res[f"idx/{i}/n_track_queries"] = np.array(len(t["track_query_boxes"]))
    sub = {k: v for k, v in gold.items() if k in res}
    assert "loss_total" in sub and any(k.startswith("idx/") for k in sub)
    df.check(res, sub, rtol=5e-3, rel_atol=2e-3)
    assert step.track_captures == 2                                # previous frame + one padded current frame


def test_graphed_tracking_steps_across_buckets_match_the_eager_route(cuda_device, strict_fp32):
    from trackformer_b200.train_step import TrainStep
    model, criterion = df.build(True, False, device=str(cuda_device), **SMALL)
    mf.canonical_weights_(model, 1)
    model.to(cuda_device).train()
    criterion.to(cuda_device).train()
    ref = copy.deepcopy(model)
    frames, _ = track_batch(0, cuda_device, sizes=((96, 128), (96, 128)), n_boxes=9)
    step = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames, track_bucket=4)
    eager = TrainStep(ref, criterion, None, use_graphs=False, track_bucket=4)
    buckets = set()
    for i in range(6):
        frames_i, targets = track_batch(20 + i, cuda_device, sizes=((96, 128), (96, 128)), n_boxes=9)
        ref_targets = copy.deepcopy(targets)
        torch.manual_seed(300 + i)
        loss = step(frames_i, targets)
        torch.manual_seed(300 + i)
        want = eager._tracking_eager(frames_i, ref_targets, None)
        for ta, tb in zip(targets, ref_targets):
            for key in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask"):
                assert torch.equal(ta[key].cpu(), tb[key].cpu()), key
        k = len(targets[0]["track_query_boxes"])
        buckets.add(-(-k // 4) * 4)
        torch.testing.assert_close(loss, want.detach(), rtol=1e-4, atol=1e-6)
        scale = float(eager.flat_grad.abs().max())
        torch.testing.assert_close(step.flat_grad, eager.flat_grad, rtol=1e-3, atol=1e-5 * scale)
    assert len(buckets) >= 2, buckets
    assert step.track_captures == 1 + len(buckets)
