"""Case runners for two-stage Deformable DETR (test infrastructure).

The same functions drive the REFERENCE (tests/golden/make_golden_two_stage.py, CPU) and the product (the tests), as
model_fixtures.py does for the one-stage model: canonical weights, seeded images and targets.  ``build(tracking,
multi_frame, **overrides)`` returns (model, criterion).  ``probe(model)`` (generator only) installs hooks and returns a
function that yields extra arrays after the forward.

The selection a model made is recorded as ``torch.topk`` of the encoder's class-0 logits, the reference's own call; the
gaps around the k-th logit show how far the fixture is from a tie.
"""
from __future__ import annotations

import numpy as np
import torch

import model_fixtures as mf

GRAD_KEYS = (
    "transformer.enc_output.weight",
    "transformer.pos_trans.weight",
    "transformer.enc_output_norm.weight",
    "class_embed.6.bias",
    "bbox_embed.6.layers.2.bias",
    "transformer.encoder.layers.0.self_attn.sampling_offsets.bias",
    "transformer.encoder.layers.5.linear2.bias",
    "bbox_embed.0.layers.2.bias",
)
GRAD_SAMPLE = 2048
TRAIN_STEP_SEED = 5          # the train-step fixture's seed: its k-th and (k+1)-th encoder logits lie >= 1e-3 apart


def sample_rows(n_tokens: int) -> np.ndarray:
    """Token rows recorded from the [B, S, .] encoder outputs: the first and last 8 (padding sits at the end of a level)
    and 48 spread over the rest."""
    spread = np.linspace(0, n_tokens - 1, 48).round().astype(np.int64)
    return np.unique(np.concatenate([np.arange(min(8, n_tokens)), spread, np.arange(max(0, n_tokens - 8), n_tokens)]))


def _np(x):
    return x.detach().cpu().numpy().copy()


def record_encoder(out, k):
    """selected tokens, gaps and sampled rows of ``out["enc_outputs"]``"""
    enc = out["enc_outputs"]
    logits0 = enc["pred_logits"][..., 0].detach().float().cpu()
    n_tok = logits0.shape[1]
    vals, sel = torch.topk(logits0, min(k + 1, n_tok), dim=1)
    rows = sample_rows(n_tok)
    res = {"selected": _np(sel[:, :k]), "rows": rows,
           "enc_logits_rows": _np(enc["pred_logits"][:, rows]), "enc_boxes_rows": _np(enc["pred_boxes"][:, rows]),
           "enc_logit0": _np(logits0)}
    if vals.shape[1] > k:
        res["boundary_gap"] = _np(vals[:, k - 1] - vals[:, k])
    res["min_adjacent_gap"] = _np((vals[:, :k - 1] - vals[:, 1:k]).min(1).values)
    return res


def _own_selection(model, res):
    """the product's own record of its selection (the decoder's row r is token ``model_selected[:, r]``)"""
    sel = getattr(model.transformer, "selected_tokens", None)
    if sel is not None:
        res["model_selected"] = _np(sel)


def run_detection(build, sizes, device="cpu", seed=0, masks=False, probe=None, **overrides):
    model, _ = build(False, False, two_stage=True, masks=masks, **overrides)
    mf.canonical_weights_(model, seed)
    model.to(device).eval()
    collect = probe(model) if probe is not None else None
    imgs = mf.make_images(seed + 1, sizes, device)
    with torch.no_grad():
        out, _, _, memory, hs = model(imgs if len(imgs) > 1 else imgs[0][None])
    k = out["pred_logits"].shape[1]
    res = {"pred_logits": _np(out["pred_logits"]), "pred_boxes": _np(out["pred_boxes"]),
           "aux0_boxes": _np(out["aux_outputs"][0]["pred_boxes"]), "aux0_logits": _np(out["aux_outputs"][0]["pred_logits"]),
           "hs_last_mean": _np(out["hs_embed"].mean(-1)), "image_digest": mf.tensor_digest(imgs[0])}
    if masks:
        res["pred_masks_mean"] = _np(out["pred_masks"].mean((-1, -2)))
    res.update(record_encoder(out, k))
    _own_selection(model, res)
    if collect is not None:
        res.update(collect())
    return res


def run_train_step(build, sizes, n_boxes, device="cpu", seed=0, probe=None, **overrides):
    """One forward + criterion + backward at dropout 0 (train mode), losses including ``_enc`` and gradient samples."""
    model, criterion = build(False, False, two_stage=True, dropout=0.0, **overrides)
    mf.canonical_weights_(model, seed)
    model.to(device).train()
    criterion.to(device).train()
    collect = probe(model) if probe is not None else None
    imgs = mf.make_images(seed + 3, sizes, device)
    targets = mf.make_targets(seed + 4, len(sizes), n_boxes, 1, device)
    out, targets_out, _, _, _ = model(imgs if len(imgs) > 1 else imgs[0][None], targets)
    loss_dict = criterion(out, targets_out)
    wd = criterion.weight_dict
    total = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
    model.zero_grad(set_to_none=True)
    total.backward()
    named = dict(model.named_parameters(remove_duplicate=False))     # the heads are shared with the decoder
    res = {"loss_total": _np(total), "pred_logits": _np(out["pred_logits"]), "pred_boxes": _np(out["pred_boxes"])}
    for k in sorted(loss_dict):
        res["loss/" + k] = _np(loss_dict[k])
    for k in GRAD_KEYS:
        g = named[k].grad
        res["grad/" + k] = _np(g.flatten()[:GRAD_SAMPLE])
        res["gradnorm/" + k] = _np(g.double().norm())
    res.update(record_encoder(out, out["pred_logits"].shape[1]))
    _own_selection(model, res)
    if collect is not None:
        res.update(collect())
    return res


def state_dict_shapes(model):
    sd = model.state_dict()
    return {"keys": np.array(list(sd)), "shapes": np.array([",".join(map(str, v.shape)) for v in sd.values()])}
