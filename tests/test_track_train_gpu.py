"""H100 tests of tracking training on the device: the forced matching cost kernel, the row-masked set loss and the
graphed tracking route of TrainStep (previous frame, device matching, bookkeeping, padded current frame from graphs).

Strict fp32 (TF32 off) unless stated; index bookkeeping bit-exact."""
import copy

import numpy as np
import pytest
import torch

import model_fixtures as mf
from conftest import load_golden
from test_model_parity_gpu import builder, check, strict_fp32  # noqa: F401  (fixture)
from test_track_train_cpu import pad_rows, random_tracking_targets, tracking_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def to(t, dev):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in t.items()}


# ---- forced matching: match_cost_track + lsa against scipy ---------------------------------------------------------
@pytest.mark.parametrize("fillers", [False, True])
def test_forced_device_matching_equals_scipy(dev, fillers):
    from trackformer_b200.matcher import HungarianMatcher
    m = HungarianMatcher(2.0, 5.0, 2.0, focal_loss=True)
    g = torch.Generator().manual_seed(3)
    nq, n_track, kb, n_layers = 40, 9, 16, 6
    targets = [random_tracking_targets(g, 7, n_track, 2, nq), random_tracking_targets(g, 12, n_track, 1, nq)]
    logits = torch.randn(n_layers, 2, n_track + nq, 20, generator=g)
    boxes = torch.rand(n_layers, 2, n_track + nq, 4, generator=g) * 0.5 + 0.1
    want = [m.forward({"pred_logits": logits[i], "pred_boxes": boxes[i]}, targets) for i in range(n_layers)]
    if fillers:
        targets = [dict(t, track_query_padding=torch.arange(kb) >= n_track) for t in targets]
        logits, boxes = pad_rows(logits, n_track, kb, 2), pad_rows(boxes, n_track, kb, 2)
    dt = [to(t, dev) for t in targets]
    src, tgt, status = m.match_layers_device(logits.to(dev), boxes.to(dev), dt, forced=True)
    assert int(status[0]) == 0
    # the kernel's cost equals the torch rewrite (same +inf pattern, finite values to fp32 rounding)
    from trackformer_b200 import ext
    tgt_ids = torch.cat([t["labels"] for t in dt])
    tgt_boxes = torch.cat([t["boxes"] for t in dt])
    pin = m.row_pin(dt, logits.shape[2], dev)
    ck = ext.load().match_cost_track(logits.to(dev), boxes.to(dev), tgt_ids, tgt_boxes, pin, 2.0, 5.0, 2.0, 0.25, 2.0)
    ct = m.force_cost(m._cost(logits.to(dev).flatten(0, 2), boxes.to(dev).flatten(0, 2), tgt_ids, tgt_boxes)
                      .view(*ck.shape), pin)
    assert torch.equal(torch.isinf(ck), torch.isinf(ct))
    fin = torch.isfinite(ct)
    torch.testing.assert_close(ck[fin], ct[fin], rtol=1e-5, atol=1e-5)
    src, tgt = src.cpu(), tgt.cpu()
    sizes = [len(t["boxes"]) for t in targets]
    for i in range(n_layers):
        ofs = 0
        for b, size in enumerate(sizes):
            s_, t_ = src[i, ofs:ofs + size], tgt[i, ofs:ofs + size] - ofs
            if fillers:
                assert not ((s_ >= n_track) & (s_ < kb)).any()
                s_ = torch.where(s_ >= kb, s_ - (kb - n_track), s_)
            ws, wt = want[i][b]
            order = torch.argsort(s_)
            assert torch.equal(s_[order], ws) and torch.equal(t_[order], wt), (i, b)
            ofs += size


# ---- row-masked set loss against fp64 torch --------------------------------------------------------------------------
def _loss_f64(logits, boxes, pairs, valid, tgt_ids, tgt_boxes, n_gt, num_boxes, alpha=0.25, gamma=2.0):
    from trackformer_b200.util import box_cxcywh_to_xyxy, paired_giou
    k_, bs, nq, c = logits.shape
    lay, bat, src, tgt = pairs
    onehot = torch.zeros(k_, bs, nq, c, dtype=torch.float64, device=logits.device)
    onehot[lay, bat, src, tgt_ids[tgt]] = 1
    p = logits.sigmoid()
    ce = torch.nn.functional.binary_cross_entropy_with_logits(logits, onehot, reduction="none")
    p_t = p * onehot + (1 - p) * (1 - onehot)
    focal = (alpha * onehot + (1 - alpha) * (1 - onehot)) * ce * (1 - p_t) ** gamma
    loss_ce = (focal * valid[None, :, :, None]).sum((1, 2, 3)) / num_boxes
    matched = boxes[lay, bat, src]
    l1 = torch.zeros(k_, dtype=torch.float64, device=logits.device).index_add(
        0, lay, (matched - tgt_boxes[tgt]).abs().sum(-1)) / num_boxes
    gi = torch.zeros(k_, dtype=torch.float64, device=logits.device).index_add(
        0, lay, 1 - paired_giou(box_cxcywh_to_xyxy(matched), box_cxcywh_to_xyxy(tgt_boxes[tgt]))) / num_boxes
    with torch.no_grad():
        n_pred = ((logits.argmax(-1) != c - 1) & valid[None].bool()).sum(2).double()
        card = (n_pred - n_gt[None]).abs().mean(1)
    return loss_ce, l1, gi, card


def test_masked_set_loss_matches_fp64(dev):
    from trackformer_b200 import ext
    g = torch.Generator().manual_seed(5)
    k_, bs, nq, c = 3, 2, 30, 20
    sizes = [4, 6]
    logits = (torch.randn(k_, bs, nq, c, generator=g) * 2).to(dev)
    boxes = (torch.rand(k_, bs, nq, 4, generator=g) * 0.5 + 0.2).to(dev)
    tgt_ids = torch.randint(0, c, (sum(sizes),), generator=g).to(dev)
    tgt_boxes = (torch.rand(sum(sizes), 4, generator=g) * 0.4 + 0.2).to(dev)
    valid = torch.ones(bs, nq, dtype=torch.bool)
    valid[0, 3:8] = False
    valid[1, 0:2] = False
    # pairs on valid rows, ascending query order per image
    src2d = torch.zeros(k_, sum(sizes), dtype=torch.int64)
    for i in range(k_):
        ofs = 0
        for b, n in enumerate(sizes):
            rows = torch.nonzero(valid[b]).flatten()
            src2d[i, ofs:ofs + n] = rows[torch.randperm(len(rows), generator=g)[:n]].sort()[0]
            ofs += n
    tgt2d = torch.stack([torch.cat([torch.randperm(n, generator=g) + sum(sizes[:b]) for b, n in enumerate(sizes)])
                         for _ in range(k_)])
    off = torch.tensor([0, sizes[0], sum(sizes)], dtype=torch.int32, device=dev)
    n_gt = torch.tensor(sizes, dtype=torch.float32, device=dev)
    nb = torch.tensor([7.0], device=dev)
    src2d, tgt2d, valid = src2d.to(dev), tgt2d.to(dev), valid.to(dev)
    out, ul, u1, ug = ext.load().set_loss_forward_masked(logits, boxes, src2d, tgt2d, tgt_ids, tgt_boxes, off, n_gt, nb,
                                                         valid.reshape(-1).to(torch.uint8), 0.25, 2.0)
    lay = torch.arange(k_, device=dev).repeat_interleave(sum(sizes))
    bat = torch.cat([torch.full((n,), b, device=dev) for b, n in enumerate(sizes)]).repeat(k_)
    lg64, bx64 = logits.double().requires_grad_(True), boxes.double().requires_grad_(True)
    ref = _loss_f64(lg64, bx64, (lay, bat, src2d.reshape(-1), tgt2d.reshape(-1)), valid.double(), tgt_ids,
                    tgt_boxes.double(), n_gt.double(), 7.0)
    for got, want in zip(out[:4], ref):
        torch.testing.assert_close(got.double(), want.detach(), rtol=2e-5, atol=1e-5)
    w = [torch.randn(k_, generator=g).to(dev) for _ in range(3)]
    gl, gb = ext.load().set_loss_backward(ul, u1, ug, w[0], w[1], w[2], nb)
    gl64, gb64 = torch.autograd.grad(sum((r * wi.double()).sum() for r, wi in zip(ref[:3], w)), (lg64, bx64))
    torch.testing.assert_close(gl.double(), gl64, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(gb.double(), gb64, rtol=1e-4, atol=1e-6)
    assert float(gl[:, ~valid].abs().max()) == 0.0 and float(gb[:, ~valid].abs().max()) == 0.0
    # an all-valid mask is the unmasked entry point, bit for bit
    a = ext.load().set_loss_forward(logits, boxes, src2d, tgt2d, tgt_ids, tgt_boxes, off, n_gt, nb, 0.25, 2.0)
    b = ext.load().set_loss_forward_masked(logits, boxes, src2d, tgt2d, tgt_ids, tgt_boxes, off, n_gt, nb,
                                           torch.ones(bs * nq, dtype=torch.uint8, device=dev), 0.25, 2.0)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---- graphed TrainStep against the reference fixture -----------------------------------------------------------------
def _fixture_setup(dev, **overrides):
    model, criterion = builder(dev)(True, False, dropout=0.0, **overrides)
    mf.canonical_weights_(model, 0)
    model.to(dev).train()
    criterion.to(dev).train()
    frames = torch.stack(mf.make_images(3, [(128, 160)], dev))
    targets = mf.make_targets(4, 1, 7, 1, dev)
    for t, pim in zip(targets, mf.make_images(5, [(128, 160)], dev)):
        pt = {k: v.clone() for k, v in t.items()}
        pt["boxes"] = (pt["boxes"] + 0.01).clamp(0.05, 0.95)
        pt["track_ids"] = torch.cat([t["track_ids"][:-1], torch.tensor([99]).to(dev)])
        t["prev_target"] = pt
        t["prev_image"] = pim
    return model, criterion, frames, targets


@pytest.mark.parametrize("bucket", [4, 6])
def test_graphed_track_step_matches_reference_fixture(dev, strict_fp32, bucket):
    from trackformer_b200.train_step import TrainStep
    gold = load_golden("train_step_tracking", "model_")
    model, criterion, frames, targets = _fixture_setup(dev)
    step = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames, track_bucket=bucket)
    torch.manual_seed(1234)
    loss = step(frames, targets)
    assert step.track_captures == 2                   # previous-frame graph + one current-frame bucket
    t = targets[0]
    assert int(gold["idx/0/n_track_queries"]) == len(t["track_query_boxes"]) == 8
    for key in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask"):
        assert np.array_equal(t[key].long().cpu().numpy(), gold[f"idx/0/{key}"]), key
    check({"loss_total": loss.cpu().numpy()}, gold, ["loss_total"])
    named = dict(model.named_parameters())
    for k in [k for k in gold if k.startswith("grad/")]:
        scale = float(np.abs(gold[k]).max())
        np.testing.assert_allclose(named[k[5:]].grad.cpu().numpy(), gold[k], rtol=5e-3,
                                   atol=2e-3 * max(scale, 1e-3), err_msg=k)


def _sequence(dev):
    """(generator seed, frames, targets) of consecutive steps with varying box counts.  With the default false-negative /
    false-positive rates the seeds give K = 8, 4, 0 (one previous frame is empty), 6 track queries, then a repeat of the
    first step (every shape warm)."""
    out = []
    for i, (n, seed) in enumerate([(7, 54), (9, 50), (5, 51), (5, 53)]):
        frames, targets = tracking_batch(20 + i, sizes=((128, 160), (128, 160)), n_boxes=n)
        if i == 2:
            targets[0]["prev_target"] = {k: v[:0] for k, v in targets[0]["prev_target"].items()}
        out.append((seed, frames.to(dev), [dict(to(t, dev), prev_target=to(t["prev_target"], dev)) for t in targets]))
    out.append(copy.deepcopy(out[0]))
    return out


def _compare_graphed_with_eager(dev, model, criterion, bucket, data, check_sync=True):
    from trackformer_b200.train_step import TrainStep
    ref_model = copy.deepcopy(model)
    graphed = TrainStep(model, criterion, None, use_graphs=True, example_frames=data[0][1], track_bucket=bucket)
    eager = TrainStep(ref_model, criterion, None, use_graphs=False, track_bucket=bucket)
    inner = graphed._track_current
    state = {"check": False, "ran": 0}

    def checked(*a, **kw):                             # the part after the bookkeeping: no host synchronisation
        if not state["check"]:
            return inner(*a, **kw)
        torch.cuda.set_sync_debug_mode("error")
        try:
            return inner(*a, **kw)
        finally:
            torch.cuda.set_sync_debug_mode("default")
            state["ran"] += 1
    graphed._track_current = checked
    ks, buckets = [], set()
    for i, (seed, frames, targets) in enumerate(data):
        ta, tb = copy.deepcopy(targets), copy.deepcopy(targets)
        state["check"] = check_sync and i == len(data) - 1
        captures = graphed.track_captures
        torch.manual_seed(seed)
        la = graphed(frames, ta)
        if state["check"]:
            assert graphed.track_captures == captures      # the repeated step replays the captured graphs
        torch.manual_seed(seed)
        lb = eager(frames, tb)
        for x, y in zip(ta, tb):
            for key in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask"):
                assert torch.equal(x[key], y[key]), (i, key)
        k = len(ta[0]["track_query_boxes"])
        ks.append(k)
        buckets.add(0 if k == 0 else -(-k // bucket))
        torch.testing.assert_close(la, lb, rtol=1e-4, atol=1e-5)
        scale = float(eager.flat_grad.abs().max())
        torch.testing.assert_close(graphed.flat_grad, eager.flat_grad, rtol=1e-3, atol=1e-4 * scale)
    if check_sync:
        assert state["ran"] == 1
    return graphed, ks, buckets


def test_graphed_steps_equal_eager_steps(dev, strict_fp32):
    model, criterion = builder(dev)(True, False, dropout=0.0, enc_layers=2, dec_layers=3, num_queries=60)
    mf.canonical_weights_(model, 0)
    model.to(dev).train()
    step, ks, buckets = _compare_graphed_with_eager(dev, model, criterion, 3, _sequence(dev))
    print("track queries per step:", ks, "buckets:", sorted(buckets), "captures:", step.track_captures)
    assert ks == [8, 4, 0, 6, 8] and buckets == {0, 2, 3}
    # one previous-frame graph + one pair per padded count seen: replays reuse them
    assert step.track_captures == 1 + len(buckets)


def test_graphed_multi_frame_model_equals_eager(dev, strict_fp32):
    model, criterion = builder(dev)(True, True, dropout=0.0)
    mf.canonical_weights_(model, 0)
    model.to(dev).train()
    data = _sequence(dev)[:2]
    step, ks, _ = _compare_graphed_with_eager(dev, model, criterion, 8, data, check_sync=False)
    print("multi-frame track queries per step:", ks)
    assert step.track_captures >= 2 and all(key[3] is not None for key in step._track_plans)
