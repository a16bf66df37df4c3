"""GPU tests of the set-criterion, Hungarian-matching and box-refinement kernels (csrc/set_loss.cu, csrc/lsa.cu,
csrc/box_refine.cu) against the REFERENCE, at the shapes training runs them.

  * fixture parity: SetCriterion.forward_stacked on the device (matching cost kernel, device Hungarian solver, fused
    loss) reproduces tests/golden/set_criterion.npz, recorded from the reference's own HungarianMatcher and
    SetCriterion in fp64 (tests/golden/make_golden_set_criterion.py): indices, per-layer losses, the box gradient and
    the logit gradient on the rows the fixture stores (every row of the last layer, every matched row).  The full
    logit gradient of all layers is pinned to the fp64 restatement by the set-loss tests below.
    The tracking case runs the forced matching, unpadded and with the track rows padded to buckets of 64 and 128.
  * set loss (set_loss_forward[_masked] + set_loss_backward) against a plain fp64 restatement of models/detr.py:213-309,
    util/misc.py:556-571 and util/box_ops.py:24-61 on the device, K = 6 layers, up to 500 + 128 queries.
  * matching cost (match_cost, match_cost_track) against models/matcher.py:70-125 elementwise.
  * the Hungarian solver (lsa) for validity and optimality against scipy on ties, integer, square, single-target,
    mixed-magnitude and forced problems, and its error return on an infeasible one.
  * refine_boxes against util/misc.py:515-519 in fp64 at the clamp gates.

Every tolerance is relative to the largest magnitude of the reference tensor it checks, with no absolute floor, and
each family carries a check that a plausible wrong variant misses the reference by far more than its tolerance.
Inputs avoid exact coordinate ties and exact arg-max ties: there the kernels and torch pick different (measure-zero)
subgradients and maxima.
"""
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

import set_criterion_fixtures as scf
from conftest import load_golden

pytestmark = pytest.mark.gpu

# the GIoU of a tiny pair carries the fp32 rounding of its corners (~3e-5 of its width): ~3e-6 of a layer's loss
LOSS_TOL = 2e-5
GRAD_LOGITS_TOL = 1e-5
GRAD_BOXES_TOL = 1e-5
# tiny boxes (w, h ~ 1e-3): their corners cx -+ w/2 carry fp32 rounding of ~3e-5 of the width, and the GIoU gradient
# scales with 1 / width; the rows matched to them are checked on their own scale at this tolerance
GRAD_TINY_TOL = 3e-4
# -log(1 - p + 1e-8) at logits +3...+8 magnifies the fp32 rounding of p: ~1e-5 of the cost's scale in fp32
COST_TOL = 5e-5
REFINE_TOL, REFINE_GRAD_TOL = 1e-6, 1e-5
LSA_REL = 1e-12
EPS32 = float(np.float32(1e-5))          # inverse_sigmoid's eps as the fp32 reference compares against it (1e-5f < 1e-5)


@pytest.fixture(scope="module")
def dev(cuda_device):
    yield cuda_device
    # release what this module allocated with its work finished, so nothing of it is freed during a later test's
    # CUDA-graph capture
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _rel_err(got, ref) -> float:
    """max |got - ref| over max |ref|."""
    ref = torch.as_tensor(ref).detach().double()
    got = torch.as_tensor(got).detach().double().to(ref.device)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    scale = float(ref.abs().max())
    assert scale > 0.0
    return float((got - ref).abs().max()) / scale


def _check(got, ref, tol, what):
    err = _rel_err(got, ref)
    assert err <= tol, f"{what}: max |error| = {err:.3e} of the reference's scale (tolerance {tol:g})"


def _check_class_error(got, ref, what):
    """class_error is a percentage (it may be 0): its scale is 100"""
    err = abs(float(got) - float(ref)) / 100.0
    assert err <= LOSS_TOL, f"{what}: class_error {float(got)} vs {float(ref)}"


# ---------------------------------------------------------------------------------------------------------------------
# fp64 restatements of the reference
def ref_box_xyxy(b):
    """util/box_ops.py:9-13"""
    cx, cy, w, h = b.unbind(-1)
    return torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], -1)


def ref_giou_matrix(a, g, hull=True):
    """util/box_ops.py:24-61 on xyxy boxes a [N,4], g [M,4] -> [N, M].  ``hull=False`` is the wrong variant without the
    enclosing-box term (plain IoU)."""
    area_a = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area_g = (g[:, 2] - g[:, 0]) * (g[:, 3] - g[:, 1])
    lt = torch.max(a[:, None, :2], g[:, :2])
    rb = torch.min(a[:, None, 2:], g[:, 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    union = area_a[:, None] + area_g - inter
    iou = inter / union
    if not hull:
        return iou
    lt = torch.min(a[:, None, :2], g[:, :2])
    rb = torch.max(a[:, None, 2:], g[:, 2:])
    wh = (rb - lt).clamp(min=0)
    area = wh[..., 0] * wh[..., 1]
    return iou - (area - union) / area


def ref_giou_pairs(a, g, hull=True):
    """torch.diag(generalized_box_iou(a, g)) of models/detr.py:306-308, row by row"""
    return torch.cat([torch.diag(ref_giou_matrix(a[i:i + 512], g[i:i + 512], hull)) for i in range(0, len(a), 512)])


def ref_focal(logits, onehot, alpha, gamma):
    """util/misc.py:556-563, elementwise"""
    prob = logits.sigmoid()
    ce = F.binary_cross_entropy_with_logits(logits, onehot, reduction="none")
    p_t = prob * onehot + (1 - prob) * (1 - onehot)
    loss = ce * ((1 - p_t) ** gamma)
    return (alpha * onehot + (1 - alpha) * (1 - onehot)) * loss


def ref_set_loss(logits, boxes, lay, bat, src, tgt, tgt_ids, tgt_boxes, valid, n_gt, num_boxes, variant=None):
    """SetCriterion's focal ``labels``, ``boxes`` and ``cardinality`` losses of every layer (models/detr.py:213-309)
    for stacked logits [K,B,Q,C] / boxes [K,B,Q,4] and the pairs (lay, bat, src) -> global box ``tgt``.  Rows with
    ``valid`` False are left out, as the reference leaves out rows it never had.
    variant "per_class": the focal loss normalised by the class count (mean over classes) instead of
    ``mean(1).sum() * Q`` (detr.py:247, misc.py:571); "no_hull": GIoU without the enclosing-box term."""
    K, B, Q, C = logits.shape
    onehot = torch.zeros_like(logits)
    onehot[lay, bat, src, tgt_ids[tgt]] = 1
    focal = ref_focal(logits, onehot, scf.ALPHA, scf.GAMMA) * valid[None, :, :, None]
    if variant == "per_class":
        loss_ce = focal.mean(3).sum((1, 2)) / num_boxes
    else:
        loss_ce = focal.mean(2).sum((1, 2)) / num_boxes * Q
    matched = boxes[lay, bat, src]
    zero = torch.zeros(K, dtype=logits.dtype, device=logits.device)
    loss_bbox = zero.index_add(0, lay, (matched - tgt_boxes[tgt]).abs().sum(-1)) / num_boxes
    giou = ref_giou_pairs(ref_box_xyxy(matched), ref_box_xyxy(tgt_boxes[tgt]), hull=variant != "no_hull")
    loss_giou = zero.index_add(0, lay, 1 - giou) / num_boxes
    with torch.no_grad():
        n_pred = ((logits.argmax(-1) != C - 1) & valid[None].bool()).sum(2).double()
        card = (n_pred - n_gt[None]).abs().mean(1)
        last = lay == K - 1
        hits = logits[-1][bat[last], src[last]].argmax(-1) == tgt_ids[tgt[last]]
        class_error = 100 - 100 * hits.double().mean()
    return loss_ce, loss_bbox, loss_giou, card, class_error


def ref_match_cost(logits, boxes, tgt_ids, tgt_boxes, alpha=scf.ALPHA, gamma=scf.GAMMA):
    """models/matcher.py:70-103 (focal) in the dtype of its inputs: [R, C], [R, 4] -> [R, T]"""
    out_prob = logits.sigmoid()
    neg = (1 - alpha) * (out_prob ** gamma) * (-(1 - out_prob + 1e-8).log())
    pos = alpha * ((1 - out_prob) ** gamma) * (-(out_prob + 1e-8).log())
    cost_class = pos[:, tgt_ids] - neg[:, tgt_ids]
    cost_bbox = torch.cdist(boxes, tgt_boxes, p=1)
    cost_giou = torch.cat([-ref_giou_matrix(ref_box_xyxy(boxes[i:i + 1024]), ref_box_xyxy(tgt_boxes))
                           for i in range(0, len(boxes), 1024)])
    return scf.COST_BBOX * cost_bbox + scf.COST_CLASS * cost_class + scf.COST_GIOU * cost_giou


def ref_forced_pattern(targets, Q):
    """The track-query rewrite of models/matcher.py:108-125 as a code per (image, row, global column): 0 the computed
    cost, 1 +inf, 2 the pinned -1."""
    sizes = [len(t["boxes"]) for t in targets]
    code = np.zeros((len(targets), Q, sum(sizes)), np.int8)
    for i, target in enumerate(targets):
        if "track_query_match_ids" not in target:
            continue
        prop_i = 0
        for j in range(Q):
            if target["track_queries_fal_pos_mask"][j]:
                code[i, j] = 1
            elif target["track_queries_mask"][j]:
                col = int(target["track_query_match_ids"][prop_i]) + sum(sizes[:i])
                prop_i += 1
                code[i, j] = 1
                code[i, :, col] = 1
                code[i, j, col] = 2
    return code


def ref_inverse_sigmoid(x, eps=EPS32):
    """util/misc.py:515-519"""
    x = x.clamp(min=0, max=1)
    x1 = x.clamp(min=eps)
    x2 = (1 - x).clamp(min=eps)
    return torch.log(x1 / x2)


# ---------------------------------------------------------------------------------------------------------------------
# fixture parity
def _criterion(C, tracking, dev):
    from trackformer_b200.criterion import SetCriterion
    from trackformer_b200.matcher import HungarianMatcher
    m = HungarianMatcher(scf.COST_CLASS, scf.COST_BBOX, scf.COST_GIOU, focal_loss=True, focal_alpha=scf.ALPHA,
                         focal_gamma=scf.GAMMA)
    crit = SetCriterion(C, m, {}, scf.EOS_COEF, ["labels", "boxes", "cardinality"], True, scf.ALPHA, scf.GAMMA,
                        tracking, True).to(dev)
    assert crit.device_matcher
    return crit


def _to(t, dev):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in t.items()}


def _run_device(crit, logits, boxes, targets, weights, dev):
    """forward_stacked on the device + backward of the weighted per-layer losses -> dict"""
    logits = logits.to(dev).requires_grad_(True)
    boxes = boxes.to(dev).requires_grad_(True)
    forced = any("track_query_match_ids" in t for t in targets)
    losses = crit.forward_stacked(logits, boxes, targets, track_queries=forced)
    ce, l1, gi = losses.stacked
    w = weights.to(dev, torch.float32)
    (w[0] * ce + w[1] * l1 + w[2] * gi).sum().backward()
    src, tgt, status = crit.matcher.match_layers_device(logits.detach(), boxes.detach(), targets, forced=forced)
    assert int(status[0]) == 0
    card = torch.stack([losses[f"cardinality_error_{k}"] for k in range(scf.K - 1)] + [losses["cardinality_error"]])
    return {"loss_ce": ce.detach(), "loss_bbox": l1.detach(), "loss_giou": gi.detach(), "cardinality_error": card,
            "class_error": losses["class_error"].detach(), "src": src.cpu().numpy(), "tgt": tgt.cpu().numpy(),
            "grad_logits": logits.grad, "grad_boxes": boxes.grad}


def _tiny_rows(fx, case, inp):
    """[K,B,Q] bool: rows the fixture matches to a tiny target box"""
    src, tgt = fx[f"{case}_src"], fx[f"{case}_tgt"]
    tb = torch.cat([t["boxes"] for t in inp["targets"]])
    off = np.concatenate([[0], np.cumsum(inp["sizes"])])
    bat = np.searchsorted(off, tgt, side="right") - 1
    lay = np.broadcast_to(np.arange(scf.K)[:, None], src.shape)
    tiny = (tb[:, 2] < 2e-3).numpy()[tgt]
    rows = np.zeros(inp["boxes"].shape[:3], bool)
    rows[lay[tiny], bat[tiny], src[tiny]] = True
    return torch.from_numpy(rows)


def _check_against_fixture(got, fx, case, inp, what):
    assert np.array_equal(got["src"], fx[f"{case}_src"]), f"{what}: matched queries"
    assert np.array_equal(got["tgt"], fx[f"{case}_tgt"]), f"{what}: matched boxes"
    for key in ("loss_ce", "loss_bbox", "loss_giou"):
        _check(got[key], fx[f"{case}_{key}"], LOSS_TOL, f"{what}: {key}")
    assert np.array_equal(got["cardinality_error"].cpu().double().numpy(), fx[f"{case}_cardinality_error"]), what
    _check_class_error(got["class_error"], fx[f"{case}_class_error"], what)
    rows = fx[f"{case}_grad_logits_rows"]
    assert np.array_equal(rows, scf.grad_logits_rows(got["src"], got["tgt"], inp["sizes"], rows.shape[2])), what
    _check(got["grad_logits"].cpu()[torch.from_numpy(rows)], fx[f"{case}_grad_logits"], GRAD_LOGITS_TOL,
           f"{what}: grad logits (last layer, matched rows)")
    tiny = _tiny_rows(fx, case, inp)
    gb, ref = got["grad_boxes"].cpu(), torch.from_numpy(fx[f"{case}_grad_boxes"])
    _check(gb[~tiny], ref[~tiny], GRAD_BOXES_TOL, f"{what}: grad boxes")
    _check(gb[tiny], ref[tiny], GRAD_TINY_TOL, f"{what}: grad boxes of tiny pairs")


@pytest.fixture(scope="module")
def fixture():
    return load_golden("set_criterion", prefix="")


def _inputs(fx, case):
    inp = scf.make_case(case)
    assert scf.checksum(inp) == str(fx[f"{case}_checksum"]), "the fixture's input generator draws differently"
    return inp


def test_detection_reproduces_reference_fixture(dev, fixture):
    inp = _inputs(fixture, "det")
    crit = _criterion(inp["C"], False, dev)
    targets = [_to(t, dev) for t in inp["targets"]]
    got = _run_device(crit, inp["logits"], inp["boxes"], targets, inp["weights"], dev)
    _check_against_fixture(got, fixture, "det", inp, "det")


def _pad(x, n_track, kb, g):
    """insert kb - n_track filler rows after the track rows (dim 2); fillers get saturated logits / valid boxes"""
    K, B, _, D = x.shape
    if D == 4:
        fill = torch.cat([torch.rand(K, B, kb - n_track, 2, generator=g) * 0.8 + 0.1,
                          torch.rand(K, B, kb - n_track, 2, generator=g) * 0.3 + 0.01], -1)
    else:
        fill = torch.randn(K, B, kb - n_track, D, generator=g) * 12
    return torch.cat([x[:, :, :n_track], fill, x[:, :, n_track:]], 2)


def test_tracking_reproduces_reference_fixture_unpadded_and_padded(dev, fixture):
    inp = _inputs(fixture, "track")
    n_track = inp["n_track"]
    crit = _criterion(inp["C"], True, dev)
    targets = [_to(t, dev) for t in inp["targets"]]
    base = _run_device(crit, inp["logits"], inp["boxes"], targets, inp["weights"], dev)
    _check_against_fixture(base, fixture, "track", inp, "track")
    g = torch.Generator().manual_seed(4)
    for kb in (64, 128):
        logits, boxes = _pad(inp["logits"], n_track, kb, g), _pad(inp["boxes"], n_track, kb, g)
        padded = [dict(t, track_query_padding=(torch.arange(kb) >= n_track).to(dev)) for t in targets]
        got = _run_device(crit, logits, boxes, padded, inp["weights"], dev)
        src = got["src"]
        assert not ((src >= n_track) & (src < kb)).any(), f"bucket {kb}: a filler row was matched"
        assert np.array_equal(np.where(src >= kb, src - (kb - n_track), src), base["src"]), kb
        assert np.array_equal(got["tgt"], base["tgt"]), kb
        # the fillers add nothing and get exactly zero gradient; the real rows get the unpadded gradients bit for bit
        real = torch.ones(logits.shape[2], dtype=torch.bool, device=dev)
        real[n_track:kb] = False
        for key in ("grad_logits", "grad_boxes"):
            assert float(got[key][:, :, ~real].abs().max()) == 0.0, (kb, key)
            assert torch.equal(got[key][:, :, real], base[key]), (kb, key)
        for key in ("loss_bbox", "loss_giou", "cardinality_error", "class_error"):
            assert torch.equal(got[key], base[key]), (kb, key)          # same pairs in the same order
        _check(got["loss_ce"], base["loss_ce"], 1e-6, f"bucket {kb}: loss_ce")     # row sums regrouped


# ---------------------------------------------------------------------------------------------------------------------
# set loss against fp64, production shapes
SET_LOSS_CASES = [
    # B, Q, C, boxes per image, masked rows
    (1, 300, 91, (1,), False),
    (2, 300, 91, (20, 100), False),
    (2, 428, 20, (100, 20), True),
    (1, 628, 20, (100,), True),
    (2, 628, 91, (1, 100), True),
]
KINDS = ("disjoint", "overlap", "inside", "outside", "overflow")


def _set_loss_problem(seed, B, Q, C, sizes, masked):
    g = torch.Generator().manual_seed(seed)
    K = scf.K
    logits = -4.6 + torch.rand(K, B, Q, C, generator=g) * 2 - 1
    boxes = torch.cat([torch.rand(K, B, Q, 2, generator=g) * 0.8 + 0.1,
                       torch.rand(K, B, Q, 2, generator=g) * 0.35 + 0.05], -1)
    valid = torch.ones(B, Q, dtype=torch.bool)
    if masked:                                   # filler runs in the track bucket and one in the object rows
        for b in range(B):
            lo = 60 + 30 * b
            valid[b, lo:128] = False
            valid[b, 200 + 17 * b:213 + 17 * b] = False
        logits[:, ~valid] = torch.randn(K, int((~valid).sum()), C, generator=g) * 15     # ignored, saturated
    T = sum(sizes)
    tgt_ids = torch.randint(0, C - 1, (T,), generator=g)
    tgt_boxes = torch.cat([torch.rand(T, 2, generator=g) * 0.6 + 0.2, torch.rand(T, 2, generator=g) * 0.25 + 0.04], 1)
    tiny = torch.arange(T) % 7 == 3                   # every seventh box is tiny, its predictions too
    tgt_boxes[tiny, 2:] = torch.rand(int(tiny.sum()), 2, generator=g) * 7e-4 + 8e-4
    src2d = torch.zeros(K, T, dtype=torch.int64)
    tgt2d = torch.zeros(K, T, dtype=torch.int64)
    for k in range(K):
        ofs = 0
        for b, n in enumerate(sizes):
            rows = torch.nonzero(valid[b]).flatten()
            s = rows[torch.randperm(len(rows), generator=g)[:n]].sort()[0]
            t = torch.randperm(n, generator=g) + ofs
            src2d[k, ofs:ofs + n], tgt2d[k, ofs:ofs + n] = s, t
            for q, j in zip(s.tolist(), t.tolist()):
                kind = "tiny" if tiny[j] else KINDS[(k + j) % len(KINDS)]
                boxes[k, b, q] = scf._pair_box(g, tgt_boxes[j], kind)
                logits[k, b, q] = scf.trained_row(g, C, int(tgt_ids[j])) if (q + k) % 3 else logits[k, b, q]
            ofs += n
    # a few confidently-background rows, some on the last class (not counted by the cardinality)
    for k in range(K):
        for q in torch.randperm(Q, generator=g)[:Q // 20].tolist():
            b = q % B
            if bool((src2d[k] == q).any()):
                continue
            logits[k, b, q] = scf.trained_row(g, C, C - 1 if q % 2 else None)
    return dict(logits=logits, boxes=boxes, valid=valid, tgt_ids=tgt_ids, tgt_boxes=tgt_boxes, src2d=src2d,
                tgt2d=tgt2d, sizes=sizes, weights=torch.rand(3, K, generator=g) * 2.5 + 0.5)


@pytest.mark.parametrize("B,Q,C,sizes,masked", SET_LOSS_CASES)
def test_set_loss_against_fp64(dev, B, Q, C, sizes, masked):
    from trackformer_b200 import ext
    m = ext.load()
    p = _set_loss_problem(Q + C + sum(sizes), B, Q, C, sizes, masked)
    K, T = scf.K, sum(sizes)
    logits, boxes = p["logits"].to(dev), p["boxes"].to(dev)
    tgt_ids, tgt_boxes = p["tgt_ids"].to(dev), p["tgt_boxes"].to(dev)
    src2d, tgt2d, valid = p["src2d"].to(dev), p["tgt2d"].to(dev), p["valid"].to(dev)
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32, device=dev)
    n_gt = torch.tensor(sizes, dtype=torch.float32, device=dev)
    nb = torch.tensor([float(T)], device=dev)
    w = p["weights"].to(dev)

    def run():
        if masked:
            out, ul, u1, ug = m.set_loss_forward_masked(logits, boxes, src2d, tgt2d, tgt_ids, tgt_boxes, off, n_gt, nb,
                                                        valid.reshape(-1).to(torch.uint8), scf.ALPHA, scf.GAMMA)
        else:
            out, ul, u1, ug = m.set_loss_forward(logits, boxes, src2d, tgt2d, tgt_ids, tgt_boxes, off, n_gt, nb,
                                                 scf.ALPHA, scf.GAMMA)
        gl, gb = m.set_loss_backward(ul, u1, ug, w[0].contiguous(), w[1].contiguous(), w[2].contiguous(), nb)
        return out, gl, gb

    out, gl, gb = run()
    again = run()
    for x, y in zip((out, gl, gb), again):
        assert torch.equal(x, y), "two runs differ"

    lay = torch.arange(K, device=dev).repeat_interleave(T)
    bat = torch.cat([torch.full((n,), b, device=dev) for b, n in enumerate(sizes)]).repeat(K)
    pairs = (lay, bat, src2d.reshape(-1), tgt2d.reshape(-1))
    lg64, bx64 = logits.double().requires_grad_(True), boxes.double().requires_grad_(True)
    args = (tgt_ids, tgt_boxes.double(), valid.double(), n_gt.double(), float(T))
    ref = ref_set_loss(lg64, bx64, *pairs, *args)
    for i, name in enumerate(("loss_ce", "loss_bbox", "loss_giou")):
        _check(out[i], ref[i], LOSS_TOL, name)
    assert torch.equal(out[3].double(), ref[3]), "cardinality_error"
    _check_class_error(out[4, -1], ref[4], "set loss")
    gl64, gb64 = torch.autograd.grad(sum((r * wi.double()).sum() for r, wi in zip(ref[:3], w)), (lg64, bx64))
    _check(gl, gl64, GRAD_LOGITS_TOL, "grad logits")
    tiny = torch.zeros(K, B, Q, dtype=torch.bool, device=dev)
    tiny[pairs[0], pairs[1], pairs[2]] = tgt_boxes[pairs[3], 2] < 2e-3
    _check(gb[~tiny], gb64[~tiny], GRAD_BOXES_TOL, "grad boxes")
    if bool(tiny.any()):
        _check(gb[tiny], gb64[tiny], GRAD_TINY_TOL, "grad boxes of tiny pairs")
    if masked:
        assert float(gl[:, ~valid].abs().max()) == 0.0 and float(gb[:, ~valid].abs().max()) == 0.0

    # the nearest mistakes miss by far more than the tolerance
    with torch.no_grad():
        wrong_ce = ref_set_loss(lg64, bx64, *pairs, *args, variant="per_class")[0]
        wrong_giou = ref_set_loss(lg64, bx64, *pairs, *args, variant="no_hull")[2]
    assert _rel_err(wrong_ce, ref[0]) > 100 * LOSS_TOL
    assert _rel_err(wrong_giou, ref[2]) > 100 * LOSS_TOL


# ---------------------------------------------------------------------------------------------------------------------
# matching cost
# -log(1 - p + 1e-8) is ill-conditioned once p is within a few fp32 ulps of 1 (logit >~ 16), where the reference itself
# runs in fp32: entries whose fp32 p >= 1 - 2^-23 are compared with the fp32 restatement instead of the fp64 one
P_SATURATED = 1.0 - 2.0 ** -23


@pytest.mark.parametrize("case", ["det", "track"])
def test_match_cost_against_reference_formula(dev, fixture, case):
    from trackformer_b200 import ext
    inp = _inputs(fixture, case)
    C = inp["C"]
    logits = inp["logits"].to(dev).reshape(-1, C)
    boxes = inp["boxes"].to(dev).reshape(-1, 4)
    tgt_ids = torch.cat([t["labels"] for t in inp["targets"]]).to(dev)
    tgt_boxes = torch.cat([t["boxes"] for t in inp["targets"]]).to(dev)
    got = ext.load().match_cost(logits, boxes, tgt_ids, tgt_boxes, scf.COST_CLASS, scf.COST_BBOX, scf.COST_GIOU,
                                scf.ALPHA, scf.GAMMA)
    ref64 = ref_match_cost(logits.double(), boxes.double(), tgt_ids, tgt_boxes.double())
    ref32 = ref_match_cost(logits, boxes, tgt_ids, tgt_boxes)
    sat = logits.sigmoid()[:, tgt_ids] >= P_SATURATED
    assert 0 < int(sat.sum()) < sat.numel() // 2
    scale = float(ref64.abs().max())
    err64 = float((got.double() - ref64)[~sat].abs().max()) / scale
    err32 = float((got.double() - ref32.double())[sat].abs().max()) / scale
    assert err64 <= COST_TOL, f"match_cost vs fp64: {err64:.3e} (tolerance {COST_TOL:g})"
    assert err32 <= COST_TOL, f"match_cost vs fp32 where p rounds to 1: {err32:.3e} (tolerance {COST_TOL:g})"
    # the focal weights swapped between the two class terms is far off
    wrong = ref_match_cost(logits.double(), boxes.double(), tgt_ids, tgt_boxes.double(), alpha=1 - scf.ALPHA)
    assert float((wrong - ref64)[~sat].abs().max()) / scale > 100 * COST_TOL


@pytest.mark.parametrize("kb", [None, 64, 128])
def test_match_cost_track_pattern_and_free_rows(dev, fixture, kb):
    """match_cost_track at the tracking fixture's size (60 track rows + 300, two images, 154 boxes, 6 layers), with
    the track rows padded to a bucket of ``kb`` filler rows: the +inf / -1 pattern is the reference loop's (fillers
    are excluded rows), and every computed entry equals match_cost bit for bit."""
    from trackformer_b200 import ext
    from trackformer_b200.matcher import HungarianMatcher
    m = ext.load()
    inp = _inputs(fixture, "track")
    n_track, C = inp["n_track"], inp["C"]
    logits, boxes = inp["logits"], inp["boxes"]
    targets = [_to(t, dev) for t in inp["targets"]]
    code = ref_forced_pattern(inp["targets"], logits.shape[2])
    if kb is not None:
        g = torch.Generator().manual_seed(kb)
        logits, boxes = _pad(logits, n_track, kb, g), _pad(boxes, n_track, kb, g)
        filler = np.ones((code.shape[0], kb - n_track, code.shape[2]), np.int8)
        code = np.concatenate([code[:, :n_track], filler, code[:, n_track:]], 1)
        targets = [dict(t, track_query_padding=(torch.arange(kb) >= n_track).to(dev)) for t in targets]
    K, B, Q, _ = logits.shape
    logits, boxes = logits.to(dev), boxes.to(dev)
    tgt_ids = torch.cat([t["labels"] for t in targets])
    tgt_boxes = torch.cat([t["boxes"] for t in targets])
    pin = HungarianMatcher.row_pin(targets, Q, dev)
    got = m.match_cost_track(logits, boxes, tgt_ids, tgt_boxes, pin, scf.COST_CLASS, scf.COST_BBOX, scf.COST_GIOU,
                             scf.ALPHA, scf.GAMMA).cpu()
    free = m.match_cost(logits, boxes, tgt_ids, tgt_boxes, scf.COST_CLASS, scf.COST_BBOX, scf.COST_GIOU, scf.ALPHA,
                        scf.GAMMA).view(K, B, Q, -1).cpu()
    code = torch.from_numpy(code)[None].expand(K, -1, -1, -1)
    assert torch.equal(torch.isposinf(got), code == 1)
    assert torch.equal(got == -1, code == 2)
    assert torch.equal(got[code == 0], free[code == 0])
    assert int((code == 2).sum()) == K * sum(len(t["track_query_match_ids"]) for t in inp["targets"])


# ---------------------------------------------------------------------------------------------------------------------
# Hungarian solver
def _lsa(cost, sizes, dev):
    from trackformer_b200 import ext
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32)
    src, tgt, status = ext.load().lsa(cost.to(dev), off.to(dev), max(sizes))
    return src.cpu().numpy(), tgt.cpu().numpy(), int(status[0])


def _gap(block, s, t):
    """(total - optimum) / |optimum| of the assignment query s[i] -> target t[i], summed in fp64 over the fp32 cost"""
    total = float(block[s, t].sum())
    rows, cols = linear_sum_assignment(block)
    opt = float(block[rows, cols].sum())
    return (total - opt) / abs(opt) if opt != 0 else (0.0 if total == opt else np.inf)


def _check_lsa(cost, sizes, src, tgt, tie_free):
    """validity and optimality of every (layer, image) block; indices equal scipy's where the optimum is unique"""
    K, B, Q, _ = cost.shape
    off = np.concatenate([[0], np.cumsum(sizes)])
    for k in range(K):
        for b in range(B):
            lo, hi = off[b], off[b + 1]
            s, t = src[k, lo:hi], tgt[k, lo:hi] - lo
            assert np.array_equal(np.sort(t), np.arange(hi - lo)), (k, b, "every target once")
            assert (s >= 0).all() and (s < Q).all() and (np.diff(s) > 0).all(), (k, b, "distinct, ascending queries")
            block = cost[k, b, :, lo:hi].numpy().astype(np.float64)
            gap = _gap(block, s, t)
            assert abs(gap) <= LSA_REL, (k, b, gap)
            if tie_free:
                rows, cols = linear_sum_assignment(block)
                assert np.array_equal(s, rows) and np.array_equal(t, cols), (k, b)


def _ties(g):
    c = torch.randn(2, 2, 300, 100, generator=g)
    c[..., 30:45] = c[..., 5:20]                      # duplicated target columns within image 0 ...
    c[..., 80:95] = c[..., 55:70]                     # ... and image 1
    c[..., 200:260, :] = c[..., 100:160, :]           # duplicated query rows
    return c, (50, 50)


LSA_PROBLEMS = {
    "ties": (_ties, False),
    "integer": (lambda g: (torch.randint(0, 3, (2, 2, 300, 137), generator=g).float(), (100, 37)), False),
    "integer_square": (lambda g: (torch.randint(0, 3, (1, 1, 64, 64), generator=g).float(), (64,)), False),
    "square_64": (lambda g: (torch.randn(3, 1, 64, 64, generator=g), (64,)), True),
    "square_300": (lambda g: (torch.randn(2, 1, 300, 300, generator=g) * 3, (300,)), True),
    "single_target": (lambda g: (torch.randn(6, 2, 300, 2, generator=g), (1, 1)), True),
    "mixed_magnitudes": (lambda g: ((torch.rand(2, 2, 300, 200, generator=g) * 2 - 1).sign()
                                    * 10 ** (torch.rand(2, 2, 300, 200, generator=g) * 8 - 4), (100, 100)), True),
}


@pytest.mark.parametrize("name", list(LSA_PROBLEMS))
def test_lsa_valid_and_optimal(dev, name):
    make, tie_free = LSA_PROBLEMS[name]
    cost, sizes = make(torch.Generator().manual_seed(len(name)))
    cost = cost.contiguous()
    src, tgt, status = _lsa(cost, sizes, dev)
    assert status == 0
    _check_lsa(cost, sizes, src, tgt, tie_free)


def test_lsa_forced_structure_and_greedy_is_rejected(dev):
    """Q = 128 + 300 rows (60 track rows per image, some false positives, the rest fillers), 100 boxes per image,
    6 layers: the cost match_cost_track builds, solved on the device, against scipy on that same cost."""
    from trackformer_b200 import ext
    from trackformer_b200.matcher import HungarianMatcher
    g = torch.Generator().manual_seed(17)
    K, B, kb, n_track, n_obj, n, C = 6, 2, 128, 60, 300, 100, 20
    Q = kb + n_obj
    targets = []
    for b in range(B):
        t = {"boxes": torch.cat([torch.rand(n, 2, generator=g) * 0.7 + 0.15, torch.rand(n, 2, generator=g) * 0.2 + 0.03],
                                1), "labels": torch.randint(0, C, (n,), generator=g)}
        is_track = torch.zeros(n_track + n_obj, dtype=torch.bool)
        is_track[:n_track] = True
        fp = torch.zeros_like(is_track)
        fp[torch.randperm(n_track, generator=g)[:7 + 5 * b]] = True
        t.update(track_queries_mask=is_track, track_queries_fal_pos_mask=fp,
                 track_query_match_ids=torch.randperm(n, generator=g)[:n_track - 7 - 5 * b],
                 track_query_padding=torch.arange(kb) >= n_track)
        targets.append(_to(t, dev))
    logits = (torch.randn(K, B, Q, C, generator=g) * 3).to(dev)
    boxes = torch.cat([torch.rand(K, B, Q, 2, generator=g) * 0.8 + 0.1, torch.rand(K, B, Q, 2, generator=g) * 0.3 + 0.02],
                      -1).to(dev)
    pin = HungarianMatcher.row_pin(targets, Q, dev)
    cost = ext.load().match_cost_track(logits, boxes, torch.cat([t["labels"] for t in targets]),
                                       torch.cat([t["boxes"] for t in targets]), pin, scf.COST_CLASS, scf.COST_BBOX,
                                       scf.COST_GIOU, scf.ALPHA, scf.GAMMA).cpu()
    sizes = (n, n)
    src, tgt, status = _lsa(cost, sizes, dev)
    assert status == 0
    _check_lsa(cost, sizes, src, tgt, tie_free=True)
    pin = pin.cpu().view(B, Q).numpy()
    for k in range(K):
        for b in range(B):
            s, t = src[k, b * n:(b + 1) * n], tgt[k, b * n:(b + 1) * n]
            assert (pin[b, s] == -1).sum() + (pin[b, s] == t).sum() == n, (k, b, "pins kept, nothing excluded")
    # a greedy assignment (each box in turn takes its cheapest free query) is rejected by the same check
    block = cost[0, 0, :, :n].numpy().astype(np.float64)
    taken, picks = set(), []
    for j in range(n):
        q = next(int(q) for q in np.argsort(block[:, j], kind="stable") if int(q) not in taken)
        taken.add(q)
        picks.append((q, j))
    picks.sort()
    s, t = np.array([p[0] for p in picks]), np.array([p[1] for p in picks])
    assert np.isfinite(block[s, t]).all()
    assert _gap(block, s, t) > 1e3 * LSA_REL


def test_lsa_infeasible_forced_problem_returns_status_2(dev):
    """5 boxes but only 3 rows left free by the forcing (17 excluded rows): the solver reports status 2, where scipy
    raises."""
    from trackformer_b200 import ext
    g = torch.Generator().manual_seed(2)
    K, B, Q, C, n = 1, 1, 20, 20, 5
    logits = torch.randn(K, B, Q, C, generator=g).to(dev)
    boxes = torch.cat([torch.rand(K, B, Q, 2, generator=g) * 0.8 + 0.1, torch.rand(K, B, Q, 2, generator=g) * 0.3 + 0.02],
                      -1).to(dev)
    tgt_boxes = torch.cat([torch.rand(n, 2, generator=g) * 0.8 + 0.1, torch.rand(n, 2, generator=g) * 0.3 + 0.02],
                          1).to(dev)
    pin = torch.tensor([-1] * 3 + [-2] * (Q - 3), dtype=torch.int32, device=dev)
    cost = ext.load().match_cost_track(logits, boxes, torch.randint(0, C, (n,), generator=g).to(dev), tgt_boxes, pin,
                                       scf.COST_CLASS, scf.COST_BBOX, scf.COST_GIOU, scf.ALPHA, scf.GAMMA).cpu()
    with pytest.raises(ValueError):
        linear_sum_assignment(cost[0, 0].numpy().astype(np.float64))
    _, _, status = _lsa(cost, (n,), dev)
    assert status == 2


# ---------------------------------------------------------------------------------------------------------------------
# box refinement
REF_SPECIALS = [0.0, 1.0, EPS32, -EPS32, float(np.float32(1 - 1e-5)), 1e-6, 1 - 1e-6, 2 * EPS32, -0.3, 1.4, 0.5,
                float(np.float32(1 + 1e-5))]


@pytest.mark.parametrize("rows", [300, 428])
@pytest.mark.parametrize("ref_dim", [2, 4])
def test_refine_boxes_against_fp64(dev, ref_dim, rows):
    from trackformer_b200.util import refine_boxes
    g = torch.Generator().manual_seed(rows + ref_dim)
    B = 2
    ref = torch.rand(B, rows, ref_dim, generator=g) * 0.98 + 0.01
    flat = ref.view(-1)
    idx = torch.randperm(flat.numel(), generator=g)[:8 * len(REF_SPECIALS)]
    flat[idx] = torch.tensor(REF_SPECIALS).repeat(8)
    delta = torch.randn(B, rows, 4, generator=g) * 2
    # the special references get a delta that keeps the output away from saturation, so their gradients are large
    dview = delta[..., :ref_dim].reshape(-1)
    dview[idx] = -ref_inverse_sigmoid(flat[idx].double()).float() + torch.randn(len(idx), generator=g) * 0.5
    delta[..., :ref_dim] = dview.view(B, rows, ref_dim)
    big = torch.randperm(delta.numel(), generator=g)[:64]
    delta.view(-1)[big] = (torch.rand(64, generator=g) * 10 + 20) * torch.where(torch.arange(64) % 2 == 0, 1.0, -1.0)
    gout = torch.randn(B, rows, 4, generator=g)

    d = delta.to(dev).requires_grad_(True)
    r = ref.to(dev).requires_grad_(True)
    out = refine_boxes(d, r)
    out.backward(gout.to(dev))

    def ref_refine(eps):
        d64 = delta.double().to(dev).requires_grad_(True)
        r64 = ref.double().to(dev).requires_grad_(True)
        inv = ref_inverse_sigmoid(r64, eps)
        z = d64 + inv if ref_dim == 4 else torch.cat([d64[..., :2] + inv, d64[..., 2:]], -1)
        y = z.sigmoid()
        y.backward(gout.double().to(dev))
        return y.detach(), d64.grad, r64.grad

    y64, gd64, gr64 = ref_refine(EPS32)
    _check(out, y64, REFINE_TOL, "refine_boxes")
    _check(d.grad, gd64, REFINE_GRAD_TOL, "grad delta")
    _check(r.grad, gr64, REFINE_GRAD_TOL, "grad reference")
    # eps taken as the double 1e-5 closes the x1 clamp's gate at x = 1e-5f: the gradient there loses its 1/x term
    _, _, gr_wrong = ref_refine(1e-5)
    assert _rel_err(gr_wrong, gr64) > 100 * REFINE_GRAD_TOL
