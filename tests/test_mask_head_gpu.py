"""GPU tests of the mask-head kernels (csrc/mask_head.cu) and the segmentation models on them.

Each kernel is checked forward and backward against its torch restatement evaluated in fp64; the CUDA mask head
(split lay1, broadcast per-image operands) against the reference composition of the CPU path; the segmentation
model and the mask loss on the GPU against the same code on the CPU.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import model_fixtures as mf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


@pytest.fixture()
def strict_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _close(got, ref, rtol=1e-4, rel_atol=1e-5):
    ref = ref.double()
    scale = float(ref.detach().abs().max()) or 1.0
    torch.testing.assert_close(got.double(), ref, rtol=rtol, atol=rel_atol * scale)


def _rand(g, *shape, dev):
    return torch.randn(*shape, generator=g, dtype=torch.float64).to(dev)


# ---------------------------------------------------------------------------------------------------------------------
def test_mask_attention_joint_softmax_fwd_bwd_with_padding(dev):
    """One softmax over each query's heads x positions (MHAttentionMap, detr_segmentation.py:214), padded positions
    at zero, and dq / dk, against fp64 torch."""
    from trackformer_b200.segmentation import mask_attention
    g = torch.Generator().manual_seed(0)
    B, Q, heads, H, W = 2, 7, 8, 13, 21
    q64, k64 = _rand(g, B, Q, heads * 32, dev=dev), _rand(g, B, H * W, heads * 32, dev=dev)
    pad = torch.zeros(B, H, W, dtype=torch.bool)
    pad[0, :, 17:] = True                              # ragged batch: image 0 is narrower, image 1 shorter
    pad[1, 10:, :] = True
    pad = pad.reshape(B, H * W).to(dev)
    gout = _rand(g, B, Q, heads, H * W, dev=dev)
    scale = 32 ** -0.5

    q, k = q64.float().requires_grad_(), k64.float().requires_grad_()
    w = mask_attention(q, k, pad, heads, scale)
    (w * gout.float()).sum().backward()

    qr, kr = q64.clone().requires_grad_(), k64.clone().requires_grad_()
    logits = torch.einsum("bqnc,bpnc->bqnp", qr.view(B, Q, heads, 32) * scale, kr.view(B, H * W, heads, 32))
    logits = logits.masked_fill(pad[:, None, None, :], float("-inf"))
    wr = logits.flatten(2).softmax(-1).view_as(logits)     # one softmax over heads x positions (MHAttentionMap)
    (wr * gout).sum().backward()
    _close(w, wr)
    assert (w[0, :, :, pad[0]] == 0).all()
    _close(q.grad, qr.grad, rtol=1e-4, rel_atol=1e-4)
    _close(k.grad, kr.grad, rtol=1e-4, rel_atol=1e-4)


@pytest.mark.parametrize("C,per_image,addend", [(264, 5, True), (48, 3, False), (16, 1, False)])
def test_group_norm_relu_fwd_bwd(dev, C, per_image, addend):
    from trackformer_b200.segmentation import group_norm_relu
    g = torch.Generator().manual_seed(C)
    images, H, W = 2, 11, 19
    N = images * per_image
    gn = torch.nn.GroupNorm(8, C).to(dev)
    with torch.no_grad():
        gn.weight.copy_(_rand(g, C, dev=dev).float())
        gn.bias.copy_(_rand(g, C, dev=dev).float() * 0.5)
    x64 = _rand(g, N, C, H, W, dev=dev)
    a64 = _rand(g, images, C, H, W, dev=dev) if addend else None
    gout = _rand(g, N, C, H, W, dev=dev)

    x = x64.float().contiguous(memory_format=torch.channels_last).requires_grad_()
    a = a64.float().requires_grad_() if addend else None
    y = group_norm_relu(x, gn, a, per_image)
    (y * gout.float()).sum().backward()

    xr = x64.clone().requires_grad_()
    ar = a64.clone().requires_grad_() if addend else None
    w64, b64 = gn.weight.detach().double().requires_grad_(), gn.bias.detach().double().requires_grad_()
    s = xr + ar.repeat_interleave(per_image, 0) if addend else xr
    yr = F.relu(F.group_norm(s, 8, w64, b64, gn.eps))
    (yr * gout).sum().backward()
    _close(y, yr)
    _close(x.grad, xr.grad, rel_atol=1e-4)
    _close(gn.weight.grad, w64.grad, rel_atol=1e-4)
    _close(gn.bias.grad, b64.grad, rel_atol=1e-4)
    if addend:
        _close(a.grad, ar.grad, rel_atol=1e-4)


@pytest.mark.parametrize("hw_in,hw_out", [((13, 21), (25, 42)), ((10, 14), (20, 28)), ((7, 9), (7, 9))])
def test_upsample_add_fwd_bwd(dev, hw_in, hw_out):
    from trackformer_b200.segmentation import upsample_add
    g = torch.Generator().manual_seed(hw_in[0])
    images, per_image, C = 2, 3, 32
    x64 = _rand(g, images * per_image, C, *hw_in, dev=dev)
    a64 = _rand(g, images, C, *hw_out, dev=dev)
    gout = _rand(g, images * per_image, C, *hw_out, dev=dev)
    x, a = x64.float().requires_grad_(), a64.float().requires_grad_()
    y = upsample_add(x, a)
    (y * gout.float()).sum().backward()
    xr, ar = x64.clone().requires_grad_(), a64.clone().requires_grad_()
    yr = ar.repeat_interleave(per_image, 0) + F.interpolate(xr, size=hw_out, mode="nearest")
    (yr * gout).sum().backward()
    _close(y, yr)
    _close(x.grad, xr.grad)
    _close(a.grad, ar.grad)


def _mask_targets(seed, sizes, counts, dev):
    g = torch.Generator().manual_seed(seed)
    return [{"masks": (torch.rand(n, h, w, generator=g) > 0.55).to(dev), "labels": torch.zeros(n, dtype=torch.int64)}
            for (h, w), n in zip(sizes, counts)]


@pytest.mark.parametrize("pairs", [5, 0])
def test_mask_loss_fwd_bwd(dev, pairs):
    from trackformer_b200.criterion import mask_losses
    g = torch.Generator().manual_seed(7)
    B, Q, h, w = 2, 9, 10, 14
    targets = _mask_targets(8, [(37, 50), (41, 45)], [3, 2], dev)        # ragged targets: padding counts
    src = torch.tensor([0 * Q + 4, 0 * Q + 1, 0 * Q + 8, 1 * Q + 2, 1 * Q + 6])[:pairs]
    tgt = torch.tensor([2, 0, 1, 4, 3])[:pairs]
    logits64 = _rand(g, B, Q, h, w, dev=dev) * 2
    num_boxes = 3.0
    lp = logits64.float().requires_grad_()
    got = mask_losses(lp, src, tgt, targets, torch.tensor(num_boxes, device=dev))
    (2.0 * got["loss_mask"] + 0.5 * got["loss_dice"]).backward()

    lr = logits64.cpu().clone().requires_grad_()
    ref = mask_losses(lr, src, tgt, [{k: v.cpu() for k, v in t.items()} for t in targets], num_boxes)
    (2.0 * ref["loss_mask"] + 0.5 * ref["loss_dice"]).backward()
    for k in ("loss_mask", "loss_dice"):
        torch.testing.assert_close(got[k].double().cpu(), ref[k], rtol=1e-5, atol=1e-7)
    _close(lp.grad.cpu(), lr.grad, rel_atol=1e-5)
    if pairs == 0:
        assert float(got["loss_mask"]) == 0.0 and float(got["loss_dice"]) == 0.0 and (lp.grad == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
def test_mask_head_split_lay1_matches_concatenated_conv(dev, strict_fp32):
    """The CUDA head (per-image lay1 part + broadcast operands) against the reference composition (_expand + cat) in
    fp64 on the CPU, forward and every parameter gradient."""
    from trackformer_b200.segmentation import MaskHeadSmallConv
    torch.manual_seed(0)
    head = MaskHeadSmallConv(256 + 8, [1024, 512, 256], 256)
    g = torch.Generator().manual_seed(1)
    B, Q, H, W = 2, 6, 5, 7
    src = torch.randn(B, 256, H, W, generator=g)
    bbox_mask = torch.rand(B, Q, 8, H, W, generator=g)
    fpns = [torch.randn(B, 1024, H, W, generator=g), torch.randn(B, 512, 2 * H, 2 * W, generator=g),
            torch.randn(B, 256, 4 * H - 1, 4 * W + 1, generator=g)]
    gout = torch.randn(B * Q, 1, 4 * H - 1, 4 * W + 1, generator=g)

    ref_head = MaskHeadSmallConv(256 + 8, [1024, 512, 256], 256).double()
    ref_head.load_state_dict(head.state_dict())
    out_ref = ref_head(src.double(), bbox_mask.double(), [f.double() for f in fpns])
    (out_ref * gout.double()).sum().backward()

    head = head.to(dev)
    out = head(src.to(dev), bbox_mask.to(dev), [f.to(dev) for f in fpns])
    (out * gout.to(dev)).sum().backward()
    _close(out.cpu(), out_ref, rtol=1e-3, rel_atol=1e-4)
    ref_grads = dict(ref_head.named_parameters())
    for name, p in head.named_parameters():
        _close(p.grad.cpu(), ref_grads[name].grad, rtol=1e-3, rel_atol=1e-3)


def _oracle_msda(monkeypatch):
    from oracle.torch_ref import msda_core_torch
    import trackformer_b200.msda_module as mm

    class _OracleFn:
        @staticmethod
        def apply(value, shapes, loc, attn, step):
            return msda_core_torch(value, shapes, loc, attn)
    monkeypatch.setattr(mm, "MSDeformAttnFunction", _OracleFn)


def test_segm_model_and_loss_match_cpu(dev, strict_fp32, monkeypatch):
    """DeformableDETRSegm at 160x224 on the sm_90a kernels against the same model on the CPU (torch ops, oracle
    MSDeformAttn): pred_masks, the mask losses and the mask-head gradients of one training forward."""
    from trackformer_b200.model_factory import build_model, default_args
    torch.manual_seed(0)
    model, criterion, post = build_model(default_args(device="cpu", masks=True))
    mf.canonical_weights_(model, 0)
    model.eval()
    imgs = mf.make_images(1, [(160, 224), (128, 192)])
    targets = mf.make_targets(2, 2, 3)
    for t, (h, w) in zip(targets, [(160, 224), (128, 192)]):
        gm = torch.Generator().manual_seed(h)
        t["masks"] = torch.rand(3, h, w, generator=gm) > 0.5

    def run(m, crit, device):
        m.zero_grad()
        out, *_ = m([i.to(device) for i in imgs])
        tg = [{k: v.to(device) for k, v in t.items()} for t in targets]
        losses = crit(out, tg)
        (losses["loss_mask"] + losses["loss_dice"]).backward()
        grads = {n: p.grad.detach().cpu().clone() for n, p in m.named_parameters()
                 if n.startswith(("mask_head", "bbox_attention")) and p.grad is not None}
        return out["pred_masks"].detach().cpu(), losses, grads

    gpu_model = __import__("copy").deepcopy(model).to(dev)
    criterion_gpu = build_model(default_args(device=str(dev), masks=True))[1]
    masks_gpu, losses_gpu, grads_gpu = run(gpu_model, criterion_gpu, dev)
    _oracle_msda(monkeypatch)
    masks_cpu, losses_cpu, grads_cpu = run(model, criterion, "cpu")
    assert masks_gpu.shape == (2, 300, 40, 56)
    scale = float(masks_cpu.abs().max())
    np.testing.assert_allclose(masks_gpu.numpy(), masks_cpu.numpy(), rtol=1e-3, atol=1e-3 * scale)
    for k in ("loss_mask", "loss_dice"):
        np.testing.assert_allclose(float(losses_gpu[k]), float(losses_cpu[k]), rtol=1e-3)
    assert set(grads_gpu) == set(grads_cpu) and len(grads_cpu) == 32
    # near-uniform attention maps leave some gradients (q_linear) at ~1e-12, pure rounding noise: the absolute
    # tolerance is relative to the largest mask-head gradient
    s = max(float(gc.abs().max()) for gc in grads_cpu.values())
    for n, gc in grads_cpu.items():
        np.testing.assert_allclose(grads_gpu[n].numpy(), gc.numpy(), rtol=2e-2, atol=1e-3 * s, err_msg=n)


def test_forward_stacked_device_matcher_with_masks(dev):
    """forward_stacked(pred_masks=...) on the device-matching route (device Hungarian matching, fused box losses,
    CUDA mask loss) against forward() on the same outputs."""
    from trackformer_b200.model_factory import build_model, default_args
    torch.manual_seed(0)
    criterion = build_model(default_args(device=str(dev), masks=True))[1]
    assert criterion.device_matcher
    g = torch.Generator().manual_seed(5)
    k, b, q = 6, 2, 300
    logits = torch.randn(k, b, q, 91, generator=g).to(dev)
    boxes = (torch.rand(k, b, q, 4, generator=g) * 0.5 + 0.25).to(dev)
    masks64 = torch.randn(b, q, 10, 14, generator=g, dtype=torch.float64)
    targets = _mask_targets(6, [(40, 56), (36, 50)], [3, 2], dev)
    for t in targets:
        t["boxes"] = (torch.rand(len(t["masks"]), 4, generator=g) * 0.4 + 0.3).to(dev)
        t["labels"] = t["labels"].to(dev)
    pm_stacked = masks64.float().to(dev).requires_grad_()
    stacked = criterion.forward_stacked(logits, boxes, targets, pred_masks=pm_stacked)
    assert stacked.stacked is not None                                   # the stacked route, not the fallback
    pm_eager = masks64.float().to(dev).requires_grad_()
    out = {"pred_logits": logits[-1], "pred_boxes": boxes[-1], "pred_masks": pm_eager,
           "aux_outputs": [{"pred_logits": logits[i], "pred_boxes": boxes[i]} for i in range(k - 1)]}
    eager = criterion(out, targets)
    for key in ("loss_mask", "loss_dice", "loss_ce", "loss_bbox", "loss_giou"):
        torch.testing.assert_close(stacked[key], eager[key], rtol=1e-5, atol=1e-6)
    (stacked["loss_mask"] + stacked["loss_dice"]).backward()
    (eager["loss_mask"] + eager["loss_dice"]).backward()
    torch.testing.assert_close(pm_stacked.grad, pm_eager.grad, rtol=1e-5, atol=1e-7)
    assert int((pm_stacked.grad.flatten(2).abs().sum(-1) > 0).sum()) == 5     # only the five matched rows
