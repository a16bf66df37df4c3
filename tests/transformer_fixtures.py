"""Shared, deterministic material for the vanilla-transformer parity tests (test infrastructure).

``run_transformer(Transformer, ...)`` is applied (a) to the REFERENCE class inside the build container by
tests/golden/make_golden_transformer.py and (b) to trackformer_b200.transformer.Transformer in the tests: both build the
train.yaml geometry (hidden 256, 8 heads, FFN 2048) with ``canonical_weights_`` and feed the same seeded inputs -- a
batch of two feature maps, the second padded on the right and bottom, 28 queries of which the first 4 carry track-query
content with a zero positional part (detr.py:62-128).  Two encoder and two decoder layers keep the recorded outputs at a
few hundred KB; the state_dict contract is checked separately at the full six layers.
"""
from __future__ import annotations

import torch

from model_fixtures import canonical_weights_

D, HEADS, FFN = 256, 8, 2048
MAP_HW, VALID_HW = (7, 10), (5, 7)
N_QUERIES, N_TRACK = 28, 4
GRAD_KEYS = ("encoder.layers.0.self_attn.in_proj_bias", "encoder.layers.1.linear2.bias",
             "decoder.layers.0.multihead_attn.in_proj_bias", "decoder.layers.1.self_attn.out_proj.bias",
             "decoder.layers.1.norm3.weight", "decoder.norm.weight")


def build(transformer_cls, pre_norm, layers=2):
    torch.manual_seed(0)
    model = transformer_cls(d_model=D, nhead=HEADS, num_encoder_layers=layers, num_decoder_layers=layers,
                            dim_feedforward=FFN, dropout=0.1, normalize_before=pre_norm, return_intermediate_dec=True)
    return canonical_weights_(model, 0).eval()


def inputs(device="cpu"):
    g = torch.Generator().manual_seed(11)
    h, w = MAP_HW
    src = torch.randn(2, D, h, w, generator=g)
    pos = torch.randn(2, D, h, w, generator=g)
    mask = torch.ones(2, h, w, dtype=torch.bool)
    mask[0] = False
    mask[1, :VALID_HW[0], :VALID_HW[1]] = False
    query_embed = torch.randn(N_QUERIES, 1, D, generator=g).repeat(1, 2, 1)
    query_embed[:N_TRACK] = 0.0
    tgt = torch.zeros(N_QUERIES, 2, D)
    tgt[:N_TRACK] = torch.randn(N_TRACK, 2, D, generator=g)
    weight = torch.randn(2, 2, N_QUERIES, D, generator=g)          # loss weights on hs [layers, B, Q, D]
    return {k: v.to(device) for k, v in dict(src=src, pos=pos, mask=mask, query_embed=query_embed, tgt=tgt,
                                             weight=weight).items()}


def run_transformer(transformer_cls, pre_norm, device="cpu"):
    model = build(transformer_cls, pre_norm).to(device)
    x = inputs(device)
    tgt = x["tgt"].clone().requires_grad_(True)
    hs, hs_without_norm, memory = model(x["src"], x["mask"], x["query_embed"], x["pos"], tgt=tgt)
    (hs * x["weight"]).sum().backward()
    params = dict(model.named_parameters())
    res = {"hs": hs, "hs_without_norm_last": hs_without_norm[-1], "memory": memory, "grad_tgt": tgt.grad}
    res.update({f"grad:{k}": params[k].grad for k in GRAD_KEYS})
    return {k: v.detach().cpu().numpy() for k, v in res.items()}


def state_dict_shapes(transformer_cls, pre_norm):
    torch.manual_seed(0)
    model = transformer_cls(d_model=D, nhead=HEADS, num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=FFN,
                            dropout=0.1, normalize_before=pre_norm, return_intermediate_dec=True)
    return {k: tuple(v.shape) for k, v in model.state_dict().items()}
