"""GPU tests of the mask-head kernels (csrc/mask_head.cu) against plain fp64 restatements of the REFERENCE's formulas,
at the shapes the segmentation model runs.

test_mask_head_gpu.py checks each kernel at small sizes; this file pins them where production runs them, so the code
paths that only large shapes reach are covered:
  * MHAttentionMap (models/detr_segmentation.py:181-216): one softmax over heads x pixels per query.  The stride-16 map
    of an 800x1333 image is 50x84 = 4200 pixels; 300 object queries (more with track queries); the dk kernel tiles the
    queries by 32.
  * GroupNorm + ReLU of each mask-head stage (models/detr_segmentation.py:143-179): gn1 has 264 channels in groups of
    33 and its input is the per-query map plus the per-image lay1 term broadcast over the image's 300 queries.
  * nearest upsampling + adapter of the FPN stages along the 800x1333 chain (50x84 -> 50x84 -> 100x167 -> 200x334;
    84 -> 167 is not 2x) and the 1080x1920 chain (68x120 -> 135x240 -> 270x480).
  * loss_masks (models/detr.py:330-357, util/misc.py:522-571): 200x334 logits bilinearly upsampled to padded 800x1333
    targets, which the forward reduces in 131 chunks of 8192 pixels per matched pair.

Every tolerance is relative to the largest magnitude of the reference tensor it checks, with no absolute floor.
"""
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HEADS, HEAD_DIM = 8, 32
ATTN_TOL, ATTN_GRAD_TOL = 2e-5, 1e-4


@pytest.fixture(scope="module")
def dev(cuda_device):
    yield cuda_device
    # the production-size cases leave several GB in the caching allocator; release everything this module allocated
    # here, with its work finished, so that nothing of it is freed during a later test's CUDA-graph capture and the
    # captures' fresh private pools do not meet a device this module has filled
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture()
def strict_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _rel_err(got, ref) -> float:
    """max |got - ref| over max |ref|."""
    ref = ref.detach().double()
    got = got.detach().double().to(ref.device)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    scale = float(ref.abs().max())
    assert scale > 0.0
    return float((got - ref).abs().max()) / scale


def _check(got, ref, tol, what):
    err = _rel_err(got, ref)
    assert err <= tol, f"{what}: max |error| = {err:.3e} of the reference's scale (tolerance {tol:g})"


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------------
# MHAttentionMap
def ref_attention_logits(qp, kp, mask, heads, scale):
    """models/detr_segmentation.py:203-213 on projected q [B, Q, D] and token-major k [B, HW, D]:
    weights [B, Q, heads, HW] with -inf on padded pixels."""
    B, Q, D = qp.shape
    qh = qp.view(B, Q, heads, D // heads)
    kh = kp.view(B, kp.shape[1], heads, D // heads)
    w = torch.einsum("bqnc,bpnc->bqnp", qh * scale, kh)
    if mask is not None:
        w = w.masked_fill(mask[:, None, None, :], float("-inf"))
    return w


def ref_softmax(logits):
    """models/detr_segmentation.py:214: F.softmax(weights.flatten(2), dim=-1) -- heads and pixels together."""
    return F.softmax(logits.flatten(2), dim=-1).view_as(logits)


def per_head_softmax(logits):
    """The wrong normalisation (each head over its own pixels), to show the checks can tell the two apart."""
    return F.softmax(logits, dim=-1)


def _assert_rejects_per_head(logits, w_ref, tol):
    """The per-head answer must miss the reference by far more than the tolerance.  Its head masses (sums over pixels)
    are all 1 while the reference's sum to 1 over the heads, so they differ by at least 1 - 1/heads."""
    w_ph = per_head_softmax(logits)
    assert _rel_err(w_ph.sum(-1), w_ref.sum(-1)) > 0.5
    assert _rel_err(w_ph.sum(-1), w_ref.sum(-1)) > 100 * tol


def _check_attention(w, w_ref, what, tol=ATTN_TOL):
    _check(w, w_ref, tol, f"{what} weights")
    _check(w.sum(-1), w_ref.sum(-1), tol, f"{what} head masses")     # each head's share of the query's mass
    torch.testing.assert_close(w.double().sum((2, 3)), torch.ones(w.shape[:2], dtype=torch.float64, device=w.device),
                               rtol=0, atol=1e-5)


def _pad_mask(B, H, W, kind, dev):
    """[B, H, W] bool: image 0 unpadded; image 1 padded on the right and bottom ("ragged") or valid at one pixel."""
    pad = torch.zeros(B, H, W, dtype=torch.bool)
    if B > 1 and kind == "ragged":
        pad[1, :, max(1, (3 * W) // 5):] = True
        pad[1, max(1, (7 * H) // 10):, :] = True
    elif B > 1 and kind == "single":
        pad[1] = True
        pad[1, H // 2, W // 3] = False
    return pad.to(dev)


def _head_spread(dtype=torch.float64, dev=None):
    """Per-head factors 1, 1.5, ..., 4.5: the heads' logits get different spreads, so their softmax partition sums
    differ strongly and no head is a rescaled copy of another."""
    return (1 + 0.5 * torch.arange(HEADS, dtype=dtype, device=dev)).repeat_interleave(HEAD_DIM)


HW_SHAPES = {35: (5, 7), 256: (16, 16), 257: (1, 257), 4200: (50, 84)}
ATTN_CASES = ([(q, hw, "ragged", 1.0) for hw in HW_SHAPES for q in (1, 31, 32, 33, 300)]
              + [(33, hw, "single", 1.0) for hw in HW_SHAPES]
              + [(300, 4200, "ragged", 1e-3)])                          # near-uniform rows


@pytest.mark.parametrize("Q,HW,pad_kind,temp", ATTN_CASES,
                         ids=[f"q{q}-hw{hw}-{k}" + ("-uniform" if t < 1 else "") for q, hw, k, t in ATTN_CASES])
def test_mask_attention_op_matches_reference(dev, Q, HW, pad_kind, temp):
    """The mask_attention op (scaled q . k, padding, softmax over heads x pixels) forward and dq / dk against the fp64
    reference formula, two images, the second padded."""
    from trackformer_b200.segmentation import mask_attention
    H, W = HW_SHAPES[HW]
    B, D, scale = 2, HEADS * HEAD_DIM, HEAD_DIM ** -0.5
    g = _gen(dev, 1000 * Q + HW)
    q32 = (torch.randn(B, Q, D, generator=g, device=dev) * _head_spread(torch.float32, dev) * temp).contiguous()
    k32 = torch.randn(B, HW, D, generator=g, device=dev)
    gout = torch.randn(B, Q, HEADS, HW, generator=g, device=dev, dtype=torch.float64)
    pad = _pad_mask(B, H, W, pad_kind, dev).reshape(B, HW)

    q, k = q32.clone().requires_grad_(), k32.clone().requires_grad_()
    w = mask_attention(q, k, pad, HEADS, scale)
    (w * gout.float()).sum().backward()

    qr, kr = q32.double().requires_grad_(), k32.double().requires_grad_()
    logits = ref_attention_logits(qr, kr, pad, HEADS, scale)
    w_ref = ref_softmax(logits)
    (w_ref * gout).sum().backward()

    _check_attention(w, w_ref, "mask_attention")
    assert (w[1][:, :, pad[1]] == 0).all()
    _check(q.grad, qr.grad, ATTN_GRAD_TOL, "dq")
    _check(k.grad, kr.grad, ATTN_GRAD_TOL, "dk")
    _assert_rejects_per_head(logits.detach(), w_ref.detach(), ATTN_TOL)


def _module_on(dev, q_dim, seed, weights=None):
    from trackformer_b200.segmentation import MHAttentionMap
    torch.manual_seed(seed)
    attn = MHAttentionMap(q_dim, HEADS * HEAD_DIM, HEADS, dropout=0.0)
    with torch.no_grad():
        if weights is None:
            attn.q_linear.weight.mul_(_head_spread(torch.float32)[:, None])
            attn.q_linear.bias.normal_(0.0, 0.1)
            attn.k_linear.bias.normal_(0.0, 0.1)
        else:
            for name, v in weights.items():
                dict(attn.named_parameters())[name].copy_(torch.from_numpy(v))
    return attn.to(dev)


def _module_reference(attn, q, k_tok, mask):
    """models/detr_segmentation.py:200-216 in fp64 with the module's parameters (k_linear as the reference's 1x1 conv
    is the same product on the token-major keys); returns logits, weights and the parameter leaves."""
    params = {n: p.detach().double().requires_grad_() for n, p in attn.named_parameters()}
    qp = F.linear(q, params["q_linear.weight"], params["q_linear.bias"])
    kp = F.linear(k_tok, params["k_linear.weight"], params["k_linear.bias"])
    logits = ref_attention_logits(qp, kp, mask, attn.num_heads, attn.normalize_fact)
    return logits, ref_softmax(logits), params


def _run_module(attn, q32, k_tok32, H, W, mask, gout):
    """The module on CUDA fp32 with k as the [B, C, H, W] view of token-major memory, as DETRSegmBase passes it."""
    B = q32.shape[0]
    q, k_tok = q32.clone().requires_grad_(), k_tok32.clone().requires_grad_()
    k = k_tok.view(B, H, W, -1).permute(0, 3, 1, 2)
    attn.zero_grad()
    w = attn(q, k, mask)
    (w * gout.float()).sum().backward()
    grads = {"q": q.grad, "k": k_tok.grad}
    grads.update({n: p.grad for n, p in attn.named_parameters()})
    return w.detach().flatten(3), grads


MODULE_CASES = [(1, 1, "none"), (1, 31, "none"), (1, 32, "none"), (1, 33, "none"), (1, 300, "none"),
                (2, 300, "ragged")]


@pytest.mark.parametrize("B,Q,pad_kind", MODULE_CASES, ids=[f"b{b}-q{q}-{k}" for b, q, k in MODULE_CASES])
def test_mhattention_map_module_matches_reference(dev, strict_fp32, B, Q, pad_kind):
    """MHAttentionMap on CUDA (its projections + mask_attention) at the 800x1333 stride-16 map against the reference
    formula in fp64 with the same parameters: bbox_mask and the gradients of q, k and the four linear parameters."""
    H, W = HW_SHAPES[4200]
    D = HEADS * HEAD_DIM
    attn = _module_on(dev, D, seed=Q)
    g = _gen(dev, 7 + Q)
    q32 = torch.randn(B, Q, D, generator=g, device=dev)
    k_tok32 = torch.randn(B, H * W, D, generator=g, device=dev)
    gout = torch.randn(B, Q, HEADS, H, W, generator=g, device=dev, dtype=torch.float64)
    mask = _pad_mask(B, H, W, pad_kind, dev) if pad_kind != "none" else None

    w, grads = _run_module(attn, q32, k_tok32, H, W, mask, gout)
    qr, kr = q32.double().requires_grad_(), k_tok32.double().requires_grad_()
    logits, w_ref, params = _module_reference(attn, qr, kr, None if mask is None else mask.reshape(B, -1))
    (w_ref * gout.flatten(3)).sum().backward()

    _check_attention(w, w_ref, "MHAttentionMap")
    _check(grads["q"], qr.grad, ATTN_GRAD_TOL, "grad q")
    _check(grads["k"], kr.grad, ATTN_GRAD_TOL, "grad k")
    for n, p in params.items():
        _check(grads[n], p.grad, ATTN_GRAD_TOL, f"grad {n}")
    _assert_rejects_per_head(logits.detach(), w_ref.detach(), ATTN_TOL)


def test_mhattention_map_module_matches_reference_fixture(dev, strict_fp32):
    """MHAttentionMap on CUDA against the reference's own module recorded in fp64 (tests/golden/mhattn_map.npz: two
    images, one padded on the right and bottom, heads whose partition sums differ by far more than 2x)."""
    from conftest import load_golden
    z = load_golden("map", prefix="mhattn_")
    names = {"q_linear.weight": "q_weight", "q_linear.bias": "q_bias", "k_linear.weight": "k_weight",
             "k_linear.bias": "k_bias"}
    attn = _module_on(dev, z["q"].shape[-1], 0, {n: z[f].astype(np.float32) for n, f in names.items()})
    B, C, H, W = z["k"].shape
    q32 = torch.from_numpy(z["q"]).float().to(dev)
    k_tok32 = torch.from_numpy(z["k"]).float().to(dev).permute(0, 2, 3, 1).reshape(B, H * W, C).contiguous()
    mask = torch.from_numpy(z["mask"]).to(dev)
    gout = torch.from_numpy(z["grad_out"]).to(dev)
    w, grads = _run_module(attn, q32, k_tok32, H, W, mask, gout)

    w_ref = torch.from_numpy(z["weights"]).to(dev).flatten(3)
    head_mass = w_ref.sum(-1)
    assert float((head_mass.max(-1).values / head_mass.min(-1).values).min()) > 2.0
    # the fixture is fp64 from fp64 inputs; the GPU sees them rounded to fp32
    _check_attention(w, w_ref, "MHAttentionMap (fixture)", 1e-4)
    _check(grads["q"], torch.from_numpy(z["grad_q"]), 2e-4, "grad q")
    k_grad = torch.from_numpy(z["grad_k"]).permute(0, 2, 3, 1).reshape(B, H * W, C)
    _check(grads["k"], k_grad, 2e-4, "grad k")
    for n, f in names.items():
        _check(grads[n], torch.from_numpy(z[f"grad_{f}"]), 2e-4, f"grad {n}")
    logits, w_ref64, _ = _module_reference(attn, q32.double(), k_tok32.double(), mask.reshape(B, -1))
    _check(w_ref64, w_ref, 1e-4, "fp64 formula on the fp32-rounded inputs vs the fixture")
    _assert_rejects_per_head(logits.detach(), w_ref, ATTN_TOL)


def test_mask_attention_is_deterministic(dev):
    """Two runs of the attention kernels give bit-identical weights, dq and dk (fixed-order sums, no float atomics)."""
    from trackformer_b200.segmentation import mask_attention
    B, Q, (H, W) = 2, 300, HW_SHAPES[4200]
    g = _gen(dev, 3)
    q32 = torch.randn(B, Q, HEADS * HEAD_DIM, generator=g, device=dev) * _head_spread(torch.float32, dev)
    k32 = torch.randn(B, H * W, HEADS * HEAD_DIM, generator=g, device=dev)
    gout = torch.randn(B, Q, HEADS, H * W, generator=g, device=dev)
    pad = _pad_mask(B, H, W, "ragged", dev).reshape(B, H * W)

    def run():
        q, k = q32.clone().requires_grad_(), k32.clone().requires_grad_()
        w = mask_attention(q, k, pad, HEADS, HEAD_DIM ** -0.5)
        (w * gout).sum().backward()
        return w.detach(), q.grad, k.grad
    for a, b in zip(run(), run()):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm + ReLU: (C, H, W, images, per_image, addend) of each stage of the head on an 800x1333 image.  The fp64
# reference runs in chunks of samples (GroupNorm is per sample) so it stays below ~0.5 GB per tensor.
GN_STAGES = {
    "gn1": (264, 50, 84, 1, 300, True),
    "gn1_two_images": (264, 50, 84, 2, 24, True),
    "gn2": (128, 50, 84, 1, 300, False),
    "gn3": (64, 50, 84, 1, 300, False),
    "gn4": (32, 100, 167, 1, 300, False),
    "gn5": (16, 200, 334, 1, 300, False),
}
GN_TOL, GN_SUM_TOL = 1e-4, 5e-4        # sums over samples / queries (affine and addend gradients) get the wider one


@pytest.mark.parametrize("stage", list(GN_STAGES))
def test_group_norm_relu_matches_reference_at_stage_shapes(dev, stage):
    from trackformer_b200.segmentation import group_norm_relu
    C, H, W, images, per_image, with_addend = GN_STAGES[stage]
    N = images * per_image
    g = _gen(dev, C + H)
    gn = torch.nn.GroupNorm(8, C).to(dev)
    with torch.no_grad():
        gn.weight.copy_(torch.randn(C, generator=g, device=dev))
        gn.bias.copy_(torch.randn(C, generator=g, device=dev) * 0.5)
    cl = torch.channels_last
    x = torch.randn(N, C, H, W, generator=g, device=dev).contiguous(memory_format=cl).requires_grad_()
    a = (torch.randn(images, C, H, W, generator=g, device=dev) * 0.5).requires_grad_() if with_addend else None
    gout = torch.randn(N, C, H, W, generator=g, device=dev).contiguous(memory_format=cl)
    y = group_norm_relu(x, gn, a, per_image)
    y.backward(gout)

    w64, b64 = gn.weight.detach().double().requires_grad_(), gn.bias.detach().double().requires_grad_()
    a64 = a.detach().double().requires_grad_() if with_addend else None
    chunk = max(1, int(6e7 // (C * H * W)))
    for n0 in range(0, N, chunk):
        n1 = min(N, n0 + chunk)
        xr = x.detach()[n0:n1].double().requires_grad_()
        s = xr + a64[torch.arange(n0, n1, device=dev) // per_image] if with_addend else xr
        z = F.group_norm(s, 8, w64, b64, gn.eps)                    # models/detr_segmentation.py:146-147 etc.
        # relu(z) as z * (z > 0); where fp64 puts z within fp32 rounding of 0, the ReLU decision is the kernel's, so
        # that one flipped decision does not move the whole gradient of that element
        near = z.detach().abs() <= 2e-6 * float(z.detach().abs().max())
        assert int(near.sum()) <= max(16, near.numel() // 10 ** 4), int(near.sum())
        yr = z * torch.where(near, y.detach()[n0:n1] > 0, z.detach() > 0)
        yr.backward(gout[n0:n1].double())
        _check(y.detach()[n0:n1], yr, GN_TOL, f"{stage} y[{n0}:{n1}]")
        _check(x.grad[n0:n1], xr.grad, GN_TOL, f"{stage} dx[{n0}:{n1}]")
    _check(gn.weight.grad, w64.grad, GN_SUM_TOL, f"{stage} dgamma")
    _check(gn.bias.grad, b64.grad, GN_SUM_TOL, f"{stage} dbeta")
    if with_addend:
        _check(a.grad, a64.grad, GN_SUM_TOL, f"{stage} daddend")


# ---------------------------------------------------------------------------------------------------------------------
# nearest upsampling + adapter: (C, (Hi, Wi), (Ho, Wo)) of the FPN stages
UP_CHAIN = {
    "800x1333_s16": (128, (50, 84), (50, 84)),
    "800x1333_s8": (64, (50, 84), (100, 167)),
    "800x1333_s4": (32, (100, 167), (200, 334)),
    "1080x1920_s8": (64, (68, 120), (135, 240)),
    "1080x1920_s4": (32, (135, 240), (270, 480)),
}


@pytest.mark.parametrize("stage", list(UP_CHAIN))
def test_upsample_add_matches_reference_along_fpn_chain(dev, stage):
    from trackformer_b200.segmentation import upsample_add
    C, hw_in, hw_out = UP_CHAIN[stage]
    images, per_image = 2, 10
    g = _gen(dev, hw_out[0])
    x = torch.randn(images * per_image, C, *hw_in, generator=g, device=dev).requires_grad_()
    a = torch.randn(images, C, *hw_out, generator=g, device=dev).requires_grad_()
    gout = torch.randn(images * per_image, C, *hw_out, generator=g, device=dev, dtype=torch.float64)
    y = upsample_add(x, a)
    (y * gout.float()).sum().backward()

    xr, ar = x.detach().double().requires_grad_(), a.detach().double().requires_grad_()
    # models/detr_segmentation.py:153-156: _expand(cur_fpn, Q) + F.interpolate(x, size, mode="nearest")
    yr = ar.repeat_interleave(per_image, 0) + F.interpolate(xr, size=hw_out, mode="nearest")
    (yr * gout).sum().backward()
    _check(y, yr, 1e-6, f"{stage} out")
    _check(x.grad, xr.grad, 1e-6, f"{stage} dx")
    _check(a.grad, ar.grad, 1e-5, f"{stage} da")


# ---------------------------------------------------------------------------------------------------------------------
# loss_masks
def ref_dice_loss(inputs, targets, num_boxes):
    """util/misc.py:522-537"""
    inputs = inputs.sigmoid().flatten(1)
    numerator = 2 * (inputs * targets).sum(1)
    denominator = inputs.sum(-1) + targets.sum(-1)
    loss = 1 - (numerator + 1) / (denominator + 1)
    return loss.sum() / num_boxes


def ref_sigmoid_focal_loss(inputs, targets, num_boxes, alpha=0.25, gamma=2):
    """util/misc.py:540-571 (no query mask, reduction on)"""
    prob = inputs.sigmoid()
    ce_loss = F.binary_cross_entropy_with_logits(inputs, targets, reduction="none")
    p_t = prob * targets + (1 - prob) * (1 - targets)
    loss = ce_loss * ((1 - p_t) ** gamma)
    if alpha >= 0:
        alpha_t = alpha * targets + (1 - alpha) * (1 - targets)
        loss = alpha_t * loss
    return loss.mean(1).sum() / num_boxes


def ref_loss_masks(pred_masks, targets, pairs, num_boxes):
    """models/detr.py:330-357: the matched rows upsampled bilinearly to the padded target size, focal + dice."""
    masks = [t["masks"] for t in targets]
    h, w = max(m.shape[1] for m in masks), max(m.shape[2] for m in masks)
    padded = torch.zeros(len(masks), max(len(m) for m in masks), h, w, dtype=torch.float64, device=pred_masks.device)
    for b, m in enumerate(masks):                                    # nested_tensor_from_tensor_list
        padded[b, :m.shape[0], :m.shape[1], :m.shape[2]] = m.double()
    bi = torch.tensor([p[0] for p in pairs], dtype=torch.long)
    si = torch.tensor([p[1] for p in pairs], dtype=torch.long)
    ti = torch.tensor([p[2] for p in pairs], dtype=torch.long)
    src = F.interpolate(pred_masks[bi, si][:, None], size=(h, w), mode="bilinear", align_corners=False)
    src = src[:, 0].flatten(1)
    tgt = padded[bi, ti].flatten(1)
    return ref_sigmoid_focal_loss(src, tgt, num_boxes), ref_dice_loss(src, tgt, num_boxes)


def _blob_masks(g, n, h, w, dev):
    """n target masks of an h x w image: an ellipse each, with a sprinkle of flipped pixels."""
    yy = torch.arange(h, device=dev, dtype=torch.float32)[:, None]
    xx = torch.arange(w, device=dev, dtype=torch.float32)[None, :]
    out = []
    for _ in range(n):
        cy, cx, ry, rx = (torch.rand(4, generator=g, device=dev) * torch.tensor([h, w, h / 3, w / 3], device=dev)
                          + torch.tensor([0.0, 0.0, 4.0, 4.0], device=dev))
        m = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
        out.append(m ^ (torch.rand(h, w, generator=g, device=dev) < 0.02))
    return torch.stack(out)


LOSS_CASES = {
    # (logits h, w), [(target h, w, masks) per image], matched pairs per image
    "800x1333_multi_chunk": ((200, 334), [(800, 1333, 12), (736, 1101, 9)], (12, 8)),
    "single_chunk": ((20, 24), [(80, 96, 4), (72, 90, 3)], (3, 3)),
    "no_pairs": ((200, 334), [(800, 1333, 2), (736, 1101, 2)], (0, 0)),
}


@pytest.mark.parametrize("case", list(LOSS_CASES))
def test_mask_loss_matches_reference(dev, case):
    """loss_mask / loss_dice and the gradient of the logits against the reference's loss on F.interpolate(bilinear)
    in fp64; two images with different target sizes, so the second image's targets are zero-padded."""
    from trackformer_b200.criterion import mask_losses
    (h, w), sizes, per_image_pairs = LOSS_CASES[case]
    B, Q = 2, 300
    g = _gen(dev, h + sum(per_image_pairs))
    targets = [{"masks": _blob_masks(g, n, th, tw, dev), "labels": torch.zeros(n, dtype=torch.int64, device=dev)}
               for th, tw, n in sizes]
    pairs, ofs = [], 0                                     # (image, query row, mask of the image)
    for b, ((_, _, n), m) in enumerate(zip(sizes, per_image_pairs)):
        rows = torch.randperm(Q, generator=g, device=dev)[:m].tolist()
        tg = torch.randperm(n, generator=g, device=dev)[:m].tolist()
        pairs += [(b, r, t) for r, t in zip(rows, tg)]
    offsets = np.cumsum([0] + [n for _, _, n in sizes])
    src = torch.tensor([b * Q + r for b, r, _ in pairs], dtype=torch.long)
    tgt = torch.tensor([int(offsets[b]) + t for b, _, t in pairs], dtype=torch.long)
    num_boxes = float(max(len(pairs), 1))
    g_mask, g_dice = 1.7, 0.6

    logits32 = torch.randn(B, Q, h, w, generator=g, device=dev) * 3
    lp = logits32.clone().requires_grad_()
    got = mask_losses(lp, src, tgt, targets, torch.tensor(num_boxes, device=dev))
    (g_mask * got["loss_mask"] + g_dice * got["loss_dice"]).backward()

    if not pairs:
        assert float(got["loss_mask"]) == 0.0 and float(got["loss_dice"]) == 0.0
        assert (lp.grad == 0).all()
        return
    lr = logits32.double().requires_grad_()
    ref_mask, ref_dice = ref_loss_masks(lr, targets, pairs, num_boxes)
    (g_mask * ref_mask + g_dice * ref_dice).backward()
    _check(got["loss_mask"], ref_mask, 2e-5, "loss_mask")
    _check(got["loss_dice"], ref_dice, 2e-5, "loss_dice")
    _check(lp.grad, lr.grad, 2e-4, "d logits")
    matched = torch.zeros(B * Q, dtype=torch.bool)
    matched[src] = True
    assert (lp.grad.flatten(0, 1)[~matched.to(dev)] == 0).all()

