"""H100 tests of segmentation training on the device: the ragged-row mask-head kernels (csrc/mask_head.cu) against fp64
torch and against their uniform (per_image) twins, and the graphed ``TrainStep(masks=True)`` against the reference
composition (``model(samples, targets)`` with the all-row head, ``SetCriterion``, backward).

Strict fp32 (TF32 off) for the step comparisons; index bookkeeping bit-exact."""
import copy

import pytest
import torch
import torch.nn.functional as F

import model_fixtures as mf
from test_model_parity_gpu import builder, strict_fp32  # noqa: F401  (fixture)
from test_track_train_gpu import _sequence

pytestmark = pytest.mark.gpu

SIZES = [3, 0, 5, 1]                    # rows per image: an image without rows in the middle
HEADS, HW = 8, 37


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def offsets_of(sizes, dev):
    acc = [0]
    for n in sizes:
        acc.append(acc[-1] + n)
    return torch.tensor(acc, dtype=torch.int32, device=dev)


def image_of(sizes, dev):
    return torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes)).to(dev)


def m():
    from trackformer_b200 import ext
    return ext.load()


# ---- mask_attn -------------------------------------------------------------------------------------------------------
def _attn_f64(q, k, pad, image, scale):
    p, d = q.shape
    qh = q.view(p, HEADS, d // HEADS)
    kh = k[image].view(p, k.shape[1], HEADS, d // HEADS)
    s = torch.einsum("phc,pjhc->phj", qh, kh) * scale
    s = s.masked_fill(pad[image][:, None, :], float("-inf"))
    return F.softmax(s.flatten(1), -1).view_as(s)


def _attn_inputs(dev, sizes, seed=0):
    g = torch.Generator().manual_seed(seed)
    b, p = len(sizes), sum(sizes)
    q = torch.randn(p, HEADS * 32, generator=g).to(dev)
    k = torch.randn(b, HW, HEADS * 32, generator=g).to(dev)
    pad = torch.zeros(b, HW, dtype=torch.bool)
    pad[:, HW - 6:] = True                                   # padded keys at the tail of every image
    if b > 2:
        pad[2, 5:9] = True                                   # and a hole inside one image
    dw = torch.randn(p, HEADS, HW, generator=g).to(dev)
    return q, k, pad.to(dev), dw


def test_ragged_attention_matches_fp64(dev):
    q, k, pad, dw = _attn_inputs(dev, SIZES)
    off, image = offsets_of(SIZES, dev), image_of(SIZES, dev)
    scale = 32 ** -0.5
    w = m().mask_attn_rows_forward(q, k, pad, off, HEADS, scale)
    dq, dk = m().mask_attn_rows_backward(q, k, off, w, dw, scale)
    q64, k64 = q.double().requires_grad_(), k.double().requires_grad_()
    w64 = _attn_f64(q64, k64, pad, image, scale)
    dq64, dk64 = torch.autograd.grad(w64, (q64, k64), dw.double())
    torch.testing.assert_close(w.double(), w64.detach(), rtol=1e-5, atol=1e-7)
    assert float(w.view(-1, HEADS, HW)[:, :, HW - 6:].abs().max()) == 0.0
    torch.testing.assert_close(dq.double(), dq64, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(dk.double(), dk64, rtol=1e-4, atol=1e-6)
    assert float(dk[1].abs().max()) == 0.0                    # the image without rows
    w2 = m().mask_attn_rows_forward(q, k, pad, off, HEADS, scale)
    dq2, dk2 = m().mask_attn_rows_backward(q, k, off, w2, dw, scale)
    assert torch.equal(w, w2) and torch.equal(dq, dq2) and torch.equal(dk, dk2)


def test_ragged_attention_with_uniform_offsets_equals_per_image(dev):
    sizes = [4, 4, 4]
    q, k, pad, dw = _attn_inputs(dev, sizes, seed=1)
    off = offsets_of(sizes, dev)
    w = m().mask_attn_rows_forward(q, k, pad, off, HEADS, 0.2)
    wu = m().mask_attn_forward(q.view(3, 4, -1), k, pad, HEADS, 0.2)
    assert torch.equal(w, wu.view_as(w))
    dq, dk = m().mask_attn_rows_backward(q, k, off, w, dw, 0.2)
    dqu, dku = m().mask_attn_backward(q.view(3, 4, -1), k, wu, dw.view_as(wu), 0.2)
    assert torch.equal(dq, dqu.view_as(dq)) and torch.equal(dk, dku)


def test_ragged_attention_without_rows(dev):
    q, k, pad, _ = _attn_inputs(dev, [0, 0])
    off = offsets_of([0, 0], dev)
    w = m().mask_attn_rows_forward(q, k, pad, off, HEADS, 0.2)
    assert w.shape == (0, HEADS, HW)
    dq, dk = m().mask_attn_rows_backward(q, k, off, w, torch.zeros_like(w), 0.2)
    assert dq.shape == (0, HEADS * 32) and float(dk.abs().max()) == 0.0
    torch.cuda.synchronize()


# ---- group_norm_relu -------------------------------------------------------------------------------------------------
def _gn_inputs(dev, sizes, c=64, hw=(6, 7), seed=2):
    g = torch.Generator().manual_seed(seed)
    cl = torch.channels_last
    x = torch.randn(sum(sizes), c, *hw, generator=g).to(dev).contiguous(memory_format=cl)
    a = torch.randn(len(sizes), c, *hw, generator=g).to(dev).contiguous(memory_format=cl)
    gamma = (1 + 0.1 * torch.randn(c, generator=g)).to(dev)
    beta = (0.1 * torch.randn(c, generator=g)).to(dev)
    dy = torch.randn(sum(sizes), c, *hw, generator=g).to(dev).contiguous(memory_format=cl)
    return x, a, gamma, beta, dy


def test_ragged_group_norm_matches_fp64(dev):
    x, a, gamma, beta, dy = _gn_inputs(dev, SIZES)
    off, image = offsets_of(SIZES, dev), image_of(SIZES, dev)
    y, mean, rstd = m().group_norm_relu_rows_forward(x, a, off, gamma, beta, 8, 1e-5)
    dx, da, dg, db = m().group_norm_relu_rows_backward(dy, x, a, off, y, gamma, mean, rstd)
    ins = [t.double().requires_grad_() for t in (x, a, gamma, beta)]
    y64 = F.relu(F.group_norm(ins[0] + ins[1][image], 8, ins[2], ins[3], 1e-5))
    want = torch.autograd.grad(y64, ins, dy.double())
    torch.testing.assert_close(y.double(), y64.detach(), rtol=1e-5, atol=1e-5)
    for got, ref, name in zip((dx, da, dg, db), want, ("dx", "daddend", "dgamma", "dbeta")):
        torch.testing.assert_close(got.double(), ref, rtol=1e-4, atol=1e-4, msg=name)
    assert float(da[1].abs().max()) == 0.0
    y2, mean2, rstd2 = m().group_norm_relu_rows_forward(x, a, off, gamma, beta, 8, 1e-5)
    again = m().group_norm_relu_rows_backward(dy, x, a, off, y2, gamma, mean2, rstd2)
    assert torch.equal(y, y2) and all(torch.equal(u, v) for u, v in zip((dx, da, dg, db), again))


def test_ragged_group_norm_with_uniform_offsets_equals_per_image(dev):
    sizes = [5, 5]
    x, a, gamma, beta, dy = _gn_inputs(dev, sizes, seed=3)
    off = offsets_of(sizes, dev)
    y, mean, rstd = m().group_norm_relu_rows_forward(x, a, off, gamma, beta, 8, 1e-5)
    yu, meanu, rstdu = m().group_norm_relu_forward(x, a, gamma, beta, 8, 5, 1e-5)
    assert torch.equal(y, yu) and torch.equal(mean, meanu) and torch.equal(rstd, rstdu)
    got = m().group_norm_relu_rows_backward(dy, x, a, off, y, gamma, mean, rstd)
    want = m().group_norm_relu_backward(dy, x, a, yu, gamma, meanu, rstdu, 5)
    assert all(torch.equal(u, v) for u, v in zip(got, want))


def test_ragged_group_norm_without_rows(dev):
    x, a, gamma, beta, dy = _gn_inputs(dev, [0, 0, 0])
    off = offsets_of([0, 0, 0], dev)
    y, mean, rstd = m().group_norm_relu_rows_forward(x, a, off, gamma, beta, 8, 1e-5)
    dx, da, dg, db = m().group_norm_relu_rows_backward(dy, x, a, off, y, gamma, mean, rstd)
    assert y.shape[0] == 0 and dx.shape[0] == 0
    assert float(da.abs().max()) == 0.0 and float(dg.abs().max()) == 0.0 and float(db.abs().max()) == 0.0


# ---- upsample_add ----------------------------------------------------------------------------------------------------
def _up_inputs(dev, sizes, seed=4):
    g = torch.Generator().manual_seed(seed)
    cl = torch.channels_last
    x = torch.randn(sum(sizes), 32, 5, 7, generator=g).to(dev).contiguous(memory_format=cl)
    a = torch.randn(len(sizes), 32, 10, 13, generator=g).to(dev).contiguous(memory_format=cl)
    dout = torch.randn(sum(sizes), 32, 10, 13, generator=g).to(dev).contiguous(memory_format=cl)
    return x, a, dout


def test_ragged_upsample_add_matches_fp64(dev):
    x, a, dout = _up_inputs(dev, SIZES)
    off, image = offsets_of(SIZES, dev), image_of(SIZES, dev)
    out = m().upsample_add_rows_forward(x, a, off)
    dx, da = m().upsample_add_rows_backward(dout, off, 5, 7)
    x64, a64 = x.double().requires_grad_(), a.double().requires_grad_()
    o64 = a64[image] + F.interpolate(x64, size=(10, 13), mode="nearest")
    dx64, da64 = torch.autograd.grad(o64, (x64, a64), dout.double())
    torch.testing.assert_close(out.double(), o64.detach(), rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(dx.double(), dx64, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(da.double(), da64, rtol=1e-5, atol=1e-5)
    assert float(da[1].abs().max()) == 0.0
    again = m().upsample_add_rows_backward(dout, off, 5, 7)
    assert torch.equal(dx, again[0]) and torch.equal(da, again[1])
    sizes = [3, 3]                                                  # uniform offsets: the per_image entry points
    x, a, dout = _up_inputs(dev, sizes, seed=5)
    off = offsets_of(sizes, dev)
    assert torch.equal(m().upsample_add_rows_forward(x, a, off), m().upsample_add_forward(x, a))
    got, want = m().upsample_add_rows_backward(dout, off, 5, 7), m().upsample_add_backward(dout, 2, 5, 7)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    x, a, dout = _up_inputs(dev, [0, 0])
    off = offsets_of([0, 0], dev)
    assert m().upsample_add_rows_forward(x, a, off).shape[0] == 0
    dx, da = m().upsample_add_rows_backward(dout, off, 5, 7)
    assert dx.shape[0] == 0 and float(da.abs().max()) == 0.0


# ---- the graphed step ------------------------------------------------------------------------------------------------
def _with_masks(data, dev, seed=9):
    g = torch.Generator().manual_seed(seed)
    for _, frames, targets in data:
        h, w = frames.shape[-2:]
        for t in targets:
            t["masks"] = (torch.rand(len(t["boxes"]), h, w, generator=g) > 0.5).to(dev)
    return data


def _reference(model, criterion, frames, targets):
    out, targets_out, _, _, _ = model(frames, targets)
    loss_dict = criterion(out, targets_out)
    wd = criterion.weight_dict
    total = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
    model.zero_grad(set_to_none=True)
    total.backward()
    return total.detach()


def _ref_flat(step, ref):
    flat = torch.zeros_like(step.flat_grad)
    named = dict(ref.named_parameters())
    names = {id(p): n for n, p in step.model.named_parameters()}
    for p in step.params:
        o = (p.grad.data_ptr() - step.flat_grad.data_ptr()) // 4
        g = named[names[id(p)]].grad
        if g is not None:
            flat[o:o + p.numel()] = g.permute(0, 2, 3, 1).reshape(-1) if p.dim() == 4 and not p.is_contiguous() \
                else g.reshape(-1)
    return flat


def _compare_with_reference(dev, model, criterion, bucket, data):
    from trackformer_b200.train_step import TrainStep
    ref = copy.deepcopy(model)
    step = TrainStep(model, criterion, None, use_graphs=True, example_frames=data[0][1], track_bucket=bucket,
                     masks=True)
    inner = step._mask_step_replayed
    state = {"check": False, "ran": 0}

    def checked(*a, **kw):                             # the mask branch between the graphs: no host synchronisation
        if not state["check"]:                         # (earlier steps meet new shapes: the criterion's index memos)
            return inner(*a, **kw)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            return inner(*a, **kw)
        finally:
            torch.cuda.set_sync_debug_mode("default")
            state["ran"] += 1
    step._mask_step_replayed = checked
    ks, buckets, captures = [], set(), []
    for i, (seed, frames, targets) in enumerate(data):
        ta, tb = copy.deepcopy(targets), copy.deepcopy(targets)
        state["check"] = i == len(data) - 1           # a repeat of the first step: every shape warm
        torch.manual_seed(seed)
        la = step(frames, ta)
        captures.append(step.track_captures)
        torch.manual_seed(seed)
        lb = _reference(ref, criterion, frames, tb)
        for x, y in zip(ta, tb):
            for key in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask"):
                assert torch.equal(x[key], y[key]), key
        k = len(ta[0]["track_query_boxes"])
        ks.append(k)
        buckets.add(0 if k == 0 else -(-k // bucket))
        torch.testing.assert_close(la, lb, rtol=1e-4, atol=1e-5)
        want = _ref_flat(step, ref)
        scale = float(want.abs().max())
        torch.testing.assert_close(step.flat_grad, want, rtol=1e-3, atol=1e-4 * scale)
    assert state["ran"] == 1
    return step, ks, buckets, captures


@pytest.mark.parametrize("kind", ["deformable", "vanilla"])
def test_graphed_mask_steps_equal_the_reference_composition(dev, strict_fp32, kind):
    if kind == "deformable":
        model, criterion = builder(dev)(True, False, dropout=0.0, masks=True, enc_layers=2, dec_layers=3,
                                        num_queries=60)
    else:
        import detr_fixtures as df
        model, criterion = df.build(True, False, device=str(dev), dropout=0.0, masks=True, enc_layers=2, dec_layers=3,
                                    num_queries=30)
    mf.canonical_weights_(model, 0)
    model.to(dev).train()
    criterion.to(dev).train()
    step, ks, buckets, captures = _compare_with_reference(dev, model, criterion, 3, _with_masks(_sequence(dev), dev))
    print(kind, "track queries per step:", ks, "captures:", captures)
    assert len(set(ks)) >= 3                                          # the track counts (and GT counts) change
    # one previous-frame graph + one pair per padded count seen; GT counts never capture
    assert step.track_captures == 1 + len(buckets)
    assert captures[-1] == captures[-2]                               # the repeated first step replays


def test_graphed_freeze_detr_step_trains_only_the_mask_head(dev, strict_fp32):
    model, criterion = builder(dev)(True, False, dropout=0.0, masks=True, freeze_detr=True, enc_layers=1,
                                    dec_layers=2, num_queries=40)
    mf.canonical_weights_(model, 1)
    model.to(dev).train()
    criterion.to(dev).train()
    seq = _with_masks(_sequence(dev), dev, seed=3)
    data = seq[:2] + seq[-1:]                                         # the last one repeats the first
    step, _, _, _ = _compare_with_reference(dev, model, criterion, 4, data)
    names = {id(p): n for n, p in model.named_parameters()}
    assert {names[id(p)].split(".")[0] for p in step.params} == {"mask_head", "bbox_attention"}
    assert float(step.flat_grad.abs().max()) > 0
    assert all(plan["g_bwd"] is None for plan in step._track_plans.values())   # nothing upstream to differentiate


def test_graphed_detection_mask_step_equals_the_reference_composition(dev, strict_fp32):
    from trackformer_b200.train_step import TrainStep
    model, criterion = builder(dev)(False, False, dropout=0.0, masks=True, enc_layers=1, dec_layers=2, num_queries=40)
    mf.canonical_weights_(model, 2)
    model.to(dev).train()
    criterion.to(dev).train()
    ref = copy.deepcopy(model)
    frames = torch.stack(mf.make_images(6, [(128, 160), (128, 160)], dev))
    step = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames, masks=True)
    for i, n in enumerate((5, 8)):                                   # GT counts change, the graphs do not
        targets = mf.make_targets(7 + i, 2, n, 1, dev)
        _with_masks([(0, frames, targets)], dev, seed=i)
        la = step(frames, copy.deepcopy(targets))
        lb = _reference(ref, criterion, frames, copy.deepcopy(targets))
        torch.testing.assert_close(la, lb, rtol=1e-4, atol=1e-5)
        want = _ref_flat(step, ref)
        torch.testing.assert_close(step.flat_grad, want, rtol=1e-3, atol=1e-4 * float(want.abs().max()))
    assert step.g_full is None and step.track_captures == 0
