"""Two-stage Deformable DETR on the H100: the proposal and selection kernels (csrc/two_stage.cu) against their host
build, the workspace Hungarian solver (csrc/lsa.cu) against the shared-memory one and scipy, the model against fixtures
recorded from the reference, the encoder loss on the device and TrainStep's routes."""
import copy

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

import two_stage_fixtures as tf
from conftest import load_golden
from test_two_stage_cpu import EMBED_ATOL, host_lib, host_proposals, host_select, ulps  # noqa: F401

pytestmark = pytest.mark.gpu

HW_800 = [(100, 167), (50, 84), (25, 42), (13, 21)]           # 22,223 tokens
HW_1333 = [(167, 167), (84, 84), (42, 42), (21, 21)]          # 37,150: a landscape and a portrait 800x1333 padded


@pytest.fixture()
def strict_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.fixture()
def tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def ext():
    from trackformer_b200 import ext as e
    return e.load()


def level_mask(hw, valid_hw):
    """[S] padding mask of one image whose content covers valid_hw = (h, w) of the finest level"""
    parts = []
    for lvl, (h, w) in enumerate(hw):
        vh, vw = -(-valid_hw[0] // (2 ** lvl)), -(-valid_hw[1] // (2 ** lvl))
        m = np.ones((h, w), bool)
        m[:vh, :vw] = False
        parts.append(m.reshape(-1))
    return np.concatenate(parts)


# ---- kernels against the host build ---------------------------------------------------------------------------------
@pytest.mark.parametrize("hw,valid", [(HW_800, None), (HW_1333, [(100, 167), (167, 100)]),
                                      ("padded_fixture", None)])
def test_proposal_kernel_matches_host_build(cuda_device, host_lib, hw, valid):
    if hw == "padded_fixture":
        gold = load_golden("det_padded_batch", "two_stage_")
        mask, hw = gold["mask"].astype(bool), [tuple(x) for x in gold["hw"]]
    elif valid is None:
        mask = np.zeros((2, sum(h * w for h, w in hw)), bool)
    else:
        mask = np.stack([level_mask(hw, v) for v in valid])
    b, s = mask.shape
    mem = torch.randn(b, s, 256, generator=torch.Generator().manual_seed(1))
    prop_h, valid_h, masked_h = host_proposals(host_lib, mask, hw, mem.numpy())
    flat = [v for pair in hw for v in pair]
    m_dev = None if not mask.any() else torch.from_numpy(mask).to(cuda_device)
    prop, vld, masked = ext().two_stage_proposals(m_dev, mem.to(cuda_device), flat, b, cuda_device.index or 0)
    assert np.array_equal(vld.cpu().numpy(), valid_h)
    assert np.array_equal(np.isinf(prop.cpu().numpy()), np.isinf(prop_h))
    assert ulps(prop.cpu().numpy(), prop_h).max() <= 2
    assert np.array_equal(masked.cpu().numpy(), masked_h)
    # memoised geometry: proposals alone, then the row mask (forward and gradient)
    prop2, vld2, _ = ext().two_stage_proposals(m_dev, None, flat, b, cuda_device.index or 0)
    assert torch.equal(prop2, prop) and torch.equal(vld2, vld)
    assert torch.equal(ext().two_stage_mask_rows(mem.to(cuda_device), vld), masked)


def test_row_mask_takes_misaligned_views_and_checks_devices(cuda_device):
    """the float4 kernels get a 16-byte aligned copy of a view that starts 4 bytes into its storage"""
    rows, c = 1000, 256
    flat = torch.randn(rows * c + 1, device=cuda_device)
    x = flat[1:].view(rows, c)
    assert x.data_ptr() % 16 != 0
    valid = (torch.arange(rows, device=cuda_device) % 3 != 0).to(torch.uint8)
    assert torch.equal(ext().two_stage_mask_rows(x, valid), x * valid[:, None].float())
    mem = x.view(2, rows // 2, c)
    flat_hw = [10, 50]
    prop, vld, masked = ext().two_stage_proposals(None, mem, flat_hw, 2, cuda_device.index or 0)
    assert torch.equal(masked, mem * vld[..., None].float())
    with pytest.raises(RuntimeError, match="one device|flags on"):
        ext().two_stage_mask_rows(x, valid.cpu())


@pytest.mark.parametrize("hw", [HW_800, HW_1333])
def test_selection_kernel_matches_host_build(cuda_device, host_lib, hw):
    s = sum(h * w for h, w in hw)
    g = torch.Generator().manual_seed(s)
    logits = torch.randn(2, s, 4, generator=g)
    logits[:, 1000:30000 // 2:13, 0] = 2.75                       # exact ties across the boundary: lower tokens win
    logits[1, :50, 0] = 3.0
    unact = torch.randn(2, s, 4, generator=g) * 2
    unact[:, 1000:30000 // 2:13] = float("inf")                     # selected invalid tokens carry +inf boxes
    idx_h, boxes_h, ref_h, embed_h = host_select(host_lib, logits.numpy(), unact.numpy(), 300)
    from trackformer_b200.deformable_transformer import proposal_dim_t
    idx, boxes, ref, embed = ext().two_stage_select(logits.to(cuda_device), unact.to(cuda_device),
                                                    proposal_dim_t(cuda_device), 300)
    assert np.array_equal(idx.cpu().numpy(), idx_h)
    assert np.array_equal(boxes.cpu().numpy(), boxes_h)
    assert np.isinf(boxes_h).any()
    assert ulps(ref.cpu().numpy(), ref_h).max() <= 2
    assert np.abs(embed.cpu().numpy() - embed_h).max() <= EMBED_ATOL
    order = torch.sort(logits[..., 0], dim=1, descending=True, stable=True)[1][:, :300]
    assert torch.equal(idx.cpu(), order)


# ---- wide Hungarian solver --------------------------------------------------------------------------------------------
def _problem(seed, k, sizes, q):
    g = torch.Generator().manual_seed(seed)
    cost = torch.rand(k, len(sizes), q, sum(sizes), generator=g) * 10
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32)
    return cost, off


@pytest.mark.parametrize("q,sizes", [(300, [20, 100]), (2000, [300, 7]), (7000, [100, 250])])
def test_wide_solver_bit_identical_to_shared_memory_solver(cuda_device, q, sizes):
    cost, off = _problem(q, 2, sizes, q)
    cost[0, 0, :, 3] = cost[0, 0, 5, 3]                              # ties: the same tie rule must decide
    a = ext().lsa(cost.to(cuda_device), off.to(cuda_device), max(sizes))
    b = ext().lsa_wide(cost.to(cuda_device), off.to(cuda_device), max(sizes))
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert int(a[2]) == 0


@pytest.mark.parametrize("t", [1, 20, 100, 300])
def test_wide_solver_equals_scipy_at_encoder_size(cuda_device, t):
    cost, off = _problem(t, 1, [t, t], 22223)
    src, tgt, status = ext().lsa(cost.to(cuda_device), off.to(cuda_device), t)
    assert int(status) == 0
    for b in range(2):
        r, c = linear_sum_assignment(cost[0, b, :, b * t:(b + 1) * t].T.double().numpy())
        rows = np.argsort(c)
        assert np.array_equal(src[0, b * t:(b + 1) * t].cpu().numpy(), np.sort(c))
        assert np.array_equal(tgt[0, b * t:(b + 1) * t].cpu().numpy() - b * t, r[rows])


def test_wide_solver_infeasible_status_and_graph_capture(cuda_device):
    cost, off = _problem(9, 1, [5, 5], 9000)
    cost[0, 1, :, 7] = float("inf")
    _, _, status = ext().lsa(cost.to(cuda_device), off.to(cuda_device), 5)
    assert int(status) == 2
    cost, off = _problem(10, 1, [30, 12], 12000)
    c_dev, o_dev = cost.to(cuda_device), off.to(cuda_device)
    want = ext().lsa(c_dev, o_dev, 30)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ext().lsa(c_dev, o_dev, 30)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = ext().lsa(c_dev, o_dev, 30)
    c_dev.copy_(_problem(11, 1, [30, 12], 12000)[0])
    graph.replay()
    torch.cuda.synchronize()
    again = ext().lsa(c_dev, o_dev, 30)
    assert all(torch.equal(x, y) for x, y in zip(got, again))
    assert not torch.equal(got[0], want[0])


# ---- model parity --------------------------------------------------------------------------------------------------
def builder(dev):
    def build(tracking, multi_frame, **overrides):
        from trackformer_b200.model_factory import build_model, default_args
        torch.manual_seed(0)
        model, criterion, _ = build_model(default_args(tracking, multi_frame, device=str(dev), **overrides))
        return model, criterion
    return build


def paired(res, gold, key):
    """``res[key]`` rows reordered to the fixture's: decoder row r of the fixture belongs to token gold_sel[r]"""
    out = np.empty_like(gold[key])
    for b in range(gold[key].shape[0]):
        pos = {int(t): r for r, t in enumerate(res["model_selected"][b])}
        out[b] = res[key][b][[pos[int(t)] for t in gold["selected"][b]]]
    return out


def check_rows(res, gold, keys, rtol=1e-3, rel_atol=1e-3):
    for k in keys:
        g = np.asarray(gold[k])
        got = paired(res, gold, k) if k in ("pred_logits", "pred_boxes", "aux0_boxes", "aux0_logits") else res[k]
        np.testing.assert_allclose(np.asarray(got), g, rtol=rtol, atol=rel_atol * (float(np.abs(g).max()) or 1.0),
                                   err_msg=k)


CASES = [("det_mini", [(160, 224)], 0), ("det_padded_batch", [(160, 224), (128, 192)], 1),
         ("det_800x1333", [(800, 1333)], 1)]


@pytest.mark.parametrize("case,sizes,seed", CASES)
def test_model_matches_reference_strict_fp32(cuda_device, strict_fp32, case, sizes, seed):
    gold = load_golden(case, "two_stage_")
    res = tf.run_detection(builder(cuda_device), sizes, device=cuda_device, seed=seed)
    for b in range(len(sizes)):
        assert set(res["model_selected"][b].tolist()) == set(gold["selected"][b].tolist())
    check_rows(res, gold, ["pred_logits", "pred_boxes", "aux0_boxes", "aux0_logits", "enc_logits_rows",
                           "enc_boxes_rows", "enc_logit0"])


def test_model_tf32_800x1333(cuda_device, tf32):
    gold = load_golden("det_800x1333", "two_stage_")
    res = tf.run_detection(builder(cuda_device), [(800, 1333)], device=cuda_device, seed=1)
    # TF32 moves the logits by ~1e-3: only tokens that close to the k-th logit may enter or leave the selection
    logit0, sel = gold["enc_logit0"][0], gold["selected"][0]
    kth = logit0[sel[-1]]
    changed = set(res["model_selected"][0].tolist()) ^ set(sel.tolist())
    assert len(changed) <= 10 and all(abs(logit0[t] - kth) < 1e-2 for t in changed), changed
    check_rows(res, gold, ["enc_logits_rows", "enc_boxes_rows"], rtol=1e-2, rel_atol=1e-2)


def test_segmentation_model_strict_fp32(cuda_device, strict_fp32):
    gold = load_golden("segm_det_mini", "two_stage_")
    res = tf.run_detection(builder(cuda_device), [(160, 224)], device=cuda_device, masks=True)
    assert set(res["model_selected"][0].tolist()) == set(gold["selected"][0].tolist())
    check_rows(res, gold, ["pred_logits", "pred_boxes", "enc_logits_rows", "enc_boxes_rows"])


# ---- criterion -------------------------------------------------------------------------------------------------------
def test_encoder_loss_device_route_equals_host_route_and_reference(cuda_device, strict_fp32):
    gold = load_golden("train_step_det", "two_stage_")
    build = builder(cuda_device)
    seed = tf.TRAIN_STEP_SEED
    res = tf.run_train_step(build, [(160, 224), (160, 224)], 6, device=cuda_device, seed=seed)
    for k in [k for k in gold if k.startswith("loss/")]:
        np.testing.assert_allclose(res[k], gold[k], rtol=1e-3, atol=1e-4, err_msg=k)

    model, criterion = build(False, False, two_stage=True, dropout=0.0)
    import model_fixtures as mf
    mf.canonical_weights_(model, seed)
    model.to(cuda_device).train()
    imgs = mf.make_images(seed + 3, [(160, 224), (160, 224)], cuda_device)
    targets = mf.make_targets(seed + 4, 2, 6, 1, cuda_device)
    out = model(imgs, targets)[0]
    logits, boxes = model.stacked_heads
    enc = model.encoder_heads
    criterion.device_matcher = False
    host = criterion(out, targets)
    host_stacked = criterion.forward_stacked(logits, boxes, targets, enc_outputs=enc)
    criterion.device_matcher = True
    num_boxes = criterion.num_boxes_device(targets, cuda_device)
    criterion.forward_stacked(logits, boxes, targets, num_boxes, enc_outputs=enc)     # index memos
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        dev_stacked = criterion.forward_stacked(logits, boxes, targets, num_boxes, enc_outputs=enc)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in ("loss_ce_enc", "loss_bbox_enc", "loss_giou_enc", "cardinality_error_enc"):
        torch.testing.assert_close(host_stacked[k], host[k], rtol=1e-5, atol=1e-6, msg=k)
        torch.testing.assert_close(dev_stacked[k], host[k], rtol=1e-4, atol=1e-5, msg=k)
        np.testing.assert_allclose(host[k].item(), gold["loss/" + k], rtol=1e-3, atol=1e-4, err_msg=k)


@pytest.mark.parametrize("n_boxes", [20, 100])
def test_encoder_loss_device_route_at_800x1333_token_count(cuda_device, n_boxes):
    """forward_stacked's encoder losses with S = 22,223 tokens per image (800x1333): the device route -- match_cost, the
    workspace solver (S is past the shared-memory solver's size) and the K = 1 fused loss, no synchronise -- against the
    host route (cost copy + scipy + the loss functions) on synthetic encoder outputs."""
    from trackformer_b200.model_factory import build_model, default_args
    _, criterion, _ = build_model(default_args(device=str(cuda_device), two_stage=True))
    s = sum(h * w for h, w in HW_800)
    g = torch.Generator().manual_seed(n_boxes)
    logits = torch.randn(2, 2, 300, 91, generator=g).to(cuda_device)
    boxes = (torch.rand(2, 2, 300, 4, generator=g) * 0.8 + 0.1).to(cuda_device)
    enc = (torch.randn(2, s, 91, generator=g).to(cuda_device), (torch.rand(2, s, 4, generator=g) * 0.8 + 0.1).to(cuda_device))
    targets = [{"boxes": torch.cat([torch.rand(n_boxes, 2, generator=g) * 0.6 + 0.2,
                                    torch.rand(n_boxes, 2, generator=g) * 0.2 + 0.05], 1).to(cuda_device),
                "labels": torch.randint(0, 90, (n_boxes,), generator=g).to(cuda_device)} for _ in range(2)]
    criterion.device_matcher = False
    host = criterion.forward_stacked(logits, boxes, targets, enc_outputs=enc)
    criterion.device_matcher = True
    num_boxes = criterion.num_boxes_device(targets, cuda_device)
    criterion.forward_stacked(logits, boxes, targets, num_boxes, enc_outputs=enc)     # index memos
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        dev = criterion.forward_stacked(logits, boxes, targets, num_boxes, enc_outputs=enc)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in ("loss_ce_enc", "loss_bbox_enc", "loss_giou_enc", "cardinality_error_enc"):
        torch.testing.assert_close(dev[k], host[k], rtol=1e-4, atol=1e-5, msg=k)


# ---- TrainStep -------------------------------------------------------------------------------------------------------
def small_model(dev):
    from trackformer_b200.model_factory import build_model, default_args
    torch.manual_seed(0)
    model, criterion, _ = build_model(default_args(device=str(dev), enc_layers=2, dec_layers=3, num_queries=50,
                                                   dropout=0.0, two_stage=True))
    return model.to(dev).train(), criterion.to(dev).train()


def targets_for(dev, seed, n):
    g = torch.Generator().manual_seed(seed)
    boxes = torch.cat([torch.rand(n, 2, generator=g) * 0.5 + 0.25, torch.rand(n, 2, generator=g) * 0.2 + 0.05], 1)
    return [{"boxes": boxes.to(dev), "labels": torch.zeros(n, dtype=torch.int64, device=dev)}]


def reference_step(model, criterion, frames, targets):
    """the eager reference composition: model + SetCriterion.forward + backward"""
    model.zero_grad(set_to_none=True)
    out = model(frames, targets)[0]
    loss_dict = criterion(out, targets)
    wd = criterion.weight_dict
    loss = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
    loss.backward()
    assert "loss_ce_enc" in loss_dict
    grads = torch.cat([p.grad.flatten() for p in model.parameters() if p.grad is not None])
    return loss.detach(), grads


@pytest.mark.parametrize("route", ["one_graph", "two_graphs", "eager"])
def test_train_step_routes_equal_reference_composition(cuda_device, strict_fp32, route):
    from trackformer_b200.train_step import TrainStep
    dev = cuda_device
    model, criterion = small_model(dev)
    model_r = copy.deepcopy(model)
    g = torch.Generator().manual_seed(7)
    frames = [torch.randn(1, 3, 192, 256, generator=g).to(dev) for _ in range(3)]
    kw = {"use_graphs": route != "eager"}
    if route != "eager":
        kw["example_frames"] = frames[0]
    if route == "one_graph":
        kw["example_targets"] = targets_for(dev, 0, 5)
    step = TrainStep(model, criterion, None, **kw)
    assert (step.g_full is not None) == (route == "one_graph")
    for i, f in enumerate(frames):
        tg = targets_for(dev, 30 + i, 5)
        if route == "one_graph":
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
        try:
            loss = step(f, tg).clone()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        loss_r, grads_r = reference_step(model_r, criterion, f, tg)
        torch.testing.assert_close(loss, loss_r, rtol=5e-3, atol=1e-4)
        grads = torch.cat([p.grad.flatten() for p, pr in zip(model.parameters(), model_r.parameters())
                           if pr.grad is not None])
        rel = float((grads - grads_r).norm() / grads_r.norm())
        assert rel < 1e-2, rel
