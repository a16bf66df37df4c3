#!/usr/bin/env python
"""MHAttentionMap golden fixture recorded FROM THE REFERENCE (build container only).

Runs the reference's own ``MHAttentionMap`` (models/detr_segmentation.py:181-216) from /root/reference/src on CPU in
fp64, imported as tests/golden/make_golden_model.py imports the reference, and stores tests/golden/mhattn_map.npz.
The module is MHAttentionMap(64, 256, 8): 8 heads of width 32 as in the model; the input width is 64 instead of 256
to keep the stored weights small.

  q [B, Q, 64], k [B, 64, H, W], mask [B, H, W]       the inputs (image 1 padded on the right and bottom)
  q_weight, q_bias, k_weight, k_bias                  the module's parameters
  grad_out [B, Q, heads, H, W]                        the seeded output gradient
  weights [B, Q, heads, H, W]                         the forward
  grad_q, grad_k, grad_q_weight, ...                  the gradients of sum(weights * grad_out)

The attention is made far from uniform on purpose: the rows of ``q_linear`` that feed head h are scaled by (1 + h),
so the heads' logits have different spreads and their softmax partition sums differ by well over 2x in every row.
A softmax normalised per head instead of over heads x pixels gives a visibly different answer on this fixture.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

B, Q, HEADS, H, W, DIM, HIDDEN = 2, 5, 8, 9, 13, 64, 256


def main():
    from make_golden_model import import_reference
    import_reference()
    from trackformer.models.detr_segmentation import MHAttentionMap

    torch.manual_seed(0)
    attn = MHAttentionMap(DIM, HIDDEN, HEADS, dropout=0.0).double()
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        head_scale = 1 + torch.arange(HEADS, dtype=torch.float64).repeat_interleave(HIDDEN // HEADS)
        attn.q_linear.weight.mul_(head_scale[:, None])
        attn.q_linear.bias.copy_(0.1 * torch.randn(HIDDEN, generator=g, dtype=torch.float64))
        attn.k_linear.bias.copy_(0.1 * torch.randn(HIDDEN, generator=g, dtype=torch.float64))
    q = torch.randn(B, Q, DIM, generator=g, dtype=torch.float64, requires_grad=True)
    k = torch.randn(B, DIM, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    mask = torch.zeros(B, H, W, dtype=torch.bool)
    mask[1, :, 10:] = True
    mask[1, 6:, :] = True
    grad_out = torch.randn(B, Q, HEADS, H, W, generator=g, dtype=torch.float64)

    weights = attn(q, k, mask)
    (weights * grad_out).sum().backward()

    z = weights.detach().flatten(3).sum(-1)                  # each head's share of the row's probability mass
    ratio = float((z.max(-1).values / z.min(-1).values).min())
    assert ratio >= 2.0, ratio
    res = {"q": q.detach(), "k": k.detach(), "mask": mask, "grad_out": grad_out, "weights": weights.detach(),
           "grad_q": q.grad, "grad_k": k.grad}
    for m in ("q", "k"):
        lin = getattr(attn, f"{m}_linear")
        res[f"{m}_weight"], res[f"{m}_bias"] = lin.weight.detach(), lin.bias.detach()
        res[f"grad_{m}_weight"], res[f"grad_{m}_bias"] = lin.weight.grad, lin.bias.grad
    path = os.path.join(HERE, "mhattn_map.npz")
    np.savez_compressed(path, **{k: v.numpy() for k, v in res.items()})
    print(f"mhattn_map -> {os.path.relpath(path)} ({os.path.getsize(path) / 1024:.0f} KiB), "
          f"min over rows of max/min head mass {ratio:.1f}", flush=True)


if __name__ == "__main__":
    main()
