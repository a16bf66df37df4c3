"""Case runners of the segmentation models, shared by the fixture recorder (tests/golden/make_golden_segm.py, which
drives the reference classes) and the parity tests (which drive trackformer_b200).

``build(tracking, multi_frame, **overrides)`` returns (model, criterion) on the CPU, as in tests/model_fixtures.py.
"""
import numpy as np
import torch

import model_fixtures as mf

SIZES = [(160, 224), (128, 192)]
ORIG_SIZES = [(80, 112), (64, 96)]
N_BOXES = 4
N_HEAD_ROWS = 8               # pred_masks rows stored in full; every row is covered by its spatial mean

# small mask-head gradients stored in full
GRAD_KEYS = tuple(f"mask_head.gn{i}.{p}" for i in range(1, 6) for p in ("weight", "bias")) + (
    "mask_head.out_lay.weight", "mask_head.out_lay.bias", "mask_head.lay5.bias", "mask_head.adapter3.bias",
    "bbox_attention.q_linear.bias", "bbox_attention.k_linear.bias")


def _to_np(x):
    return x.detach().cpu().numpy().copy()


def mask_targets(seed, sizes, n_boxes, device="cpu"):
    """Box targets of model_fixtures.make_targets plus one boolean mask per box at the image size: the box interior
    with a seeded ragged border, so matched masks overlap their predictions' support."""
    targets = mf.make_targets(seed, len(sizes), n_boxes, 1, device)
    g = torch.Generator().manual_seed(seed + 100)
    for t, (h, w) in zip(targets, sizes):
        ys = torch.arange(h, dtype=torch.float32)[:, None] / h
        xs = torch.arange(w, dtype=torch.float32)[None, :] / w
        masks = []
        for cx, cy, bw, bh in t["boxes"].cpu().tolist():
            inside = ((xs - cx).abs() <= bw / 2) & ((ys - cy).abs() <= bh / 2)
            masks.append(inside & (torch.rand(h, w, generator=g) > 0.15))
        t["masks"] = torch.stack(masks).to(device)
    return targets


def run_segm_train_step(build, postprocess_cls, device="cpu", seed=0):
    """DeformableDETRSegm on a padded two-image batch: one forward + criterion (with ``masks``) + backward, dropout
    off, then PostProcessSegm on the outputs."""
    model, criterion = build(False, False, dropout=0.0, masks=True)
    mf.canonical_weights_(model, seed)
    model.to(device).train()
    criterion.to(device).train()
    imgs = mf.make_images(seed + 3, SIZES, device)
    targets = mask_targets(seed + 4, SIZES, N_BOXES, device)
    out, targets_out, _, _, _ = model(imgs, targets)
    loss_dict = criterion(out, targets_out)
    wd = criterion.weight_dict
    total = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
    model.zero_grad(set_to_none=True)
    total.backward()
    named = dict(model.named_parameters())
    pm = out["pred_masks"]
    res = {"pred_masks_rows": _to_np(pm[:, :N_HEAD_ROWS]), "pred_masks_mean": _to_np(pm.mean((-1, -2))),
           "loss_total": _to_np(total), "loss_mask": _to_np(loss_dict["loss_mask"]),
           "loss_dice": _to_np(loss_dict["loss_dice"])}
    for k in GRAD_KEYS:
        res["grad/" + k] = _to_np(named[k].grad)
    sq = sum(float((p.grad.double() ** 2).sum()) for n, p in named.items()
             if p.grad is not None and n.startswith(("mask_head.", "bbox_attention.")))
    res["grad_mask_head_norm"] = torch.tensor(sq).sqrt().numpy()
    sq = sum(float((p.grad.double() ** 2).sum()) for p in model.parameters() if p.grad is not None)
    res["grad_global_norm"] = torch.tensor(sq).sqrt().numpy()

    keep = torch.zeros(len(SIZES), pm.shape[1], dtype=torch.bool)
    keep[:, :6] = True
    results = [{} for _ in SIZES]
    post = postprocess_cls()(results, {"pred_masks": pm.detach()}, torch.tensor(ORIG_SIZES), torch.tensor(SIZES),
                             results_mask=keep)
    for i, r in enumerate(post):
        res[f"segm/{i}"] = r["masks"].cpu().numpy()
    probs = postprocess_cls()([{} for _ in SIZES], {"pred_masks": pm.detach()}, torch.tensor(ORIG_SIZES),
                              torch.tensor(SIZES), return_probs=True, results_mask=keep)
    for i, r in enumerate(probs):
        res[f"segm_probs/{i}"] = r["masks"].cpu().numpy()
    res["state_dict_keys"] = np.array(sorted(model.state_dict()))
    return res


def run_segm_two_frames(build, device="cpu", seed=0, n_track=12):
    """DeformableDETRSegmTracking in tracking mode: frame 1 with the two-argument call, frame 2 with ``n_track``
    track queries and frame 1's features -- the three-argument call of the tracker (models/tracker.py:306)."""
    model, _ = build(True, False, masks=True)
    mf.canonical_weights_(model, seed)
    model.to(device)
    model.tracking()
    f1, f2 = mf.make_images(seed + 2, [SIZES[0], SIZES[0]], device)
    with torch.no_grad():
        out1, _, feats1, _, _ = model(f1[None])
        tgt = [{"track_query_boxes": out1["pred_boxes"][0, :n_track],
                "track_query_hs_embeds": out1["hs_embed"][0, :n_track], "image_id": torch.tensor([1]).to(device)}]
        out2, _, _, _, _ = model(f2[None], tgt, feats1)
    return {"f1_masks_rows": _to_np(out1["pred_masks"][:, :N_HEAD_ROWS]),
            "f1_masks_mean": _to_np(out1["pred_masks"].mean((-1, -2))),
            "f2_masks_rows": _to_np(out2["pred_masks"][:, :N_HEAD_ROWS + n_track]),
            "f2_masks_mean": _to_np(out2["pred_masks"].mean((-1, -2))),
            "f2_boxes": _to_np(out2["pred_boxes"]), "state_dict_keys": np.array(sorted(model.state_dict()))}
