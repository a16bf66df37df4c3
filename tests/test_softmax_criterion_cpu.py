"""CPU tests of the softmax (vanilla-DETR) route of ``SetCriterion.forward_stacked`` and of the TrainStep tracking route
it opens.  On the CPU the stacked pass is the torch restatement (host forcing, row mask, false-positive track queries
at full weight), the reference the GPU tests hold the fused kernels (csrc/set_loss.cu) to."""
import copy
import types

import numpy as np
import pytest
import torch

import detr_fixtures as df
import model_fixtures as mf
import softmax_criterion_fixtures as smf
from conftest import load_golden

SMALL = dict(enc_layers=1, dec_layers=2, num_queries=20, dropout=0.0)


def criterion_for(case, fp):
    from trackformer_b200.criterion import SetCriterion
    from trackformer_b200.matcher import HungarianMatcher
    matcher = HungarianMatcher(smf.COST_CLASS, smf.COST_BBOX, smf.COST_GIOU, focal_loss=False)
    return SetCriterion(case["C"] - 1, matcher, {}, smf.EOS_COEF, ["labels", "boxes", "cardinality"], False, 0.25, 2.0,
                        True, smf.FP_WEIGHT[fp])


def weighted_total(losses, w):
    names = ("loss_ce", "loss_bbox", "loss_giou")
    return sum(w[i, k] * losses[n if k == smf.K - 1 else f"{n}_{k}"] for i, n in enumerate(names)
               for k in range(smf.K))


def pad_rows(x, n_track, kb):
    """insert kb - n_track filler rows (random values) after the n_track track rows of dimension 2"""
    g = torch.Generator().manual_seed(kb)
    shape = (*x.shape[:2], kb - n_track, x.shape[3])
    fill = torch.rand(shape, generator=g, dtype=x.dtype) if x.shape[-1] == 4 else \
        torch.randn(shape, generator=g, dtype=x.dtype) * 3
    return torch.cat([x[:, :, :n_track], fill, x[:, :, n_track:]], 2)


@pytest.fixture(scope="module")
def gold():
    return load_golden("softmax_criterion", "")


@pytest.mark.parametrize("fp", list(smf.FP_WEIGHT))
@pytest.mark.parametrize("name", list(smf.CASES))
def test_torch_route_equals_reference_fixture(gold, name, fp):
    case = smf.make_case(name)
    pre = f"{name}_{fp}_"
    assert str(gold[pre + "checksum"]) == smf.checksum(case)
    crit = criterion_for(case, fp).double()
    logits = case["logits"].double().requires_grad_(True)
    boxes = case["boxes"].double().requires_grad_(True)
    targets = [{k: (v.double() if k == "boxes" else v) for k, v in t.items()} for t in case["targets"]]
    got = crit.forward_stacked(logits, boxes, targets, track_queries=True)
    for base in ("loss_ce", "loss_bbox", "loss_giou", "cardinality_error"):
        vals = np.array([float(got[base if k == smf.K - 1 else f"{base}_{k}"]) for k in range(smf.K)])
        np.testing.assert_allclose(vals, gold[pre + base], rtol=1e-10, atol=1e-12, err_msg=base)
    np.testing.assert_allclose(float(got["class_error"]), gold[pre + "class_error"], rtol=1e-10)
    gl, gb = torch.autograd.grad(weighted_total(got, case["weights"]), (logits, boxes))
    rows = gold[pre + "grad_logits_rows"]
    np.testing.assert_allclose(gl.numpy()[rows], gold[pre + "grad_logits"], rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(gb.numpy(), gold[pre + "grad_boxes"], rtol=1e-5, atol=1e-9)


@pytest.mark.parametrize("kb_extra", [3, 12])
@pytest.mark.parametrize("name", list(smf.CASES))
def test_filler_rows_change_nothing(name, kb_extra):
    """the track rows padded to a bucket: same losses, same gradients on the real rows, zero on the fillers"""
    case = smf.make_case(name)
    crit = criterion_for(case, "fp1")
    n_track = case["n_track"]
    kb = n_track + kb_extra
    logits = case["logits"].double().requires_grad_(True)
    boxes = case["boxes"].double().requires_grad_(True)
    targets = [{k: (v.double() if k == "boxes" else v) for k, v in t.items()} for t in case["targets"]]
    want = crit.forward_stacked(logits, boxes, targets, track_queries=True)
    gl_want, gb_want = torch.autograd.grad(weighted_total(want, case["weights"]), (logits, boxes))

    pl = pad_rows(case["logits"].double(), n_track, kb).requires_grad_(True)
    pb = pad_rows(case["boxes"].double(), n_track, kb).requires_grad_(True)
    padded = [dict(t, track_query_padding=torch.arange(kb) >= n_track) for t in targets]
    got = crit.forward_stacked(pl, pb, padded, track_queries=True)
    assert set(got) == set(want)
    for k in want:
        torch.testing.assert_close(got[k], want[k], rtol=1e-12, atol=1e-12, msg=k)
    gl, gb = torch.autograd.grad(weighted_total(got, case["weights"]), (pl, pb))
    real = torch.cat([torch.arange(n_track), torch.arange(kb, pl.shape[2])])
    torch.testing.assert_close(gl[:, :, real], gl_want, rtol=1e-10, atol=1e-14)
    torch.testing.assert_close(gb[:, :, real], gb_want, rtol=1e-10, atol=1e-14)
    assert float(gl[:, :, n_track:kb].abs().max()) == 0.0 and float(gb[:, :, n_track:kb].abs().max()) == 0.0


def test_tracking_route_admits_the_softmax_box_only_criterion():
    from trackformer_b200.model_factory import build_model, vanilla_args
    from trackformer_b200.train_step import TrainStep
    model, crit, _ = build_model(vanilla_args(tracking=True, dataset="mot", device="cpu", **SMALL))
    assert not crit.focal_loss
    model.train()
    targets = [{"prev_image": torch.zeros(3, 64, 64), "prev_target": {}}]
    route = lambda m, c, t: TrainStep._tracking_route(types.SimpleNamespace(model=m, criterion=c), t)   # noqa: E731
    assert route(model, crit, targets) == "track"
    assert route(model, crit, [dict(targets[0], prev_prev_image=torch.zeros(3, 64, 64))]) == "eager"
    model._backprop_prev_frame = True
    assert route(model, crit, targets) == "eager"
    segm, segm_crit, _ = build_model(vanilla_args(tracking=True, masks=True, dataset="mot", device="cpu", **SMALL))
    segm.train()
    assert route(segm, segm_crit, targets) == "eager"


def reference_step(model, criterion, frames, targets):
    out, targets_out, _, _, _ = model(frames, targets)
    loss_dict = criterion(out, targets_out)
    wd = criterion.weight_dict
    total = sum(loss_dict[k] * wd[k] for k in loss_dict if k in wd)
    model.zero_grad(set_to_none=True)
    total.backward()
    return total.detach(), targets_out


def flat_of(step, model):
    flat = torch.zeros_like(step.flat_grad)
    named = dict(model.named_parameters())
    names = {id(p): n for n, p in step.model.named_parameters()}
    for p in step.params:
        o = (p.grad.data_ptr() - step.flat_grad.data_ptr()) // 4
        g = named[names[id(p)]].grad
        if g is not None:
            flat[o:o + p.numel()] = g.reshape(-1) if g.is_contiguous() else g.permute(0, 2, 3, 1).reshape(-1)
    return flat


@pytest.mark.parametrize("seed", [0, 2])
def test_vanilla_tracking_train_step_equals_the_eager_model(seed):
    from trackformer_b200.train_step import TrainStep
    model, criterion = df.build(True, False, **SMALL)
    mf.canonical_weights_(model, seed)
    model.train()
    ref = copy.deepcopy(model)
    frames = torch.stack(mf.make_images(seed + 3, [(96, 128), (96, 128)]))
    targets = mf.make_targets(seed + 4, 2, 7, 1)
    for t, pim in zip(targets, mf.make_images(seed + 5, [(96, 128), (96, 128)])):
        pt = {k: v.clone() for k, v in t.items()}
        pt["boxes"] = (pt["boxes"] + 0.01).clamp(0.05, 0.95)
        pt["track_ids"] = torch.cat([t["track_ids"][:-1], torch.tensor([99])])
        t["prev_target"], t["prev_image"] = pt, pim
    ref_targets = copy.deepcopy(targets)
    step = TrainStep(model, criterion, None, use_graphs=False, track_bucket=4)
    assert step._tracking_route(targets) == "track"

    torch.manual_seed(1234)
    loss = step(frames, targets)
    torch.manual_seed(1234)
    ref_loss, ref_targets = reference_step(ref, criterion, frames, ref_targets)
    for ta, tb in zip(targets, ref_targets):
        for key in ("track_query_match_ids", "track_queries_mask", "track_queries_fal_pos_mask"):
            assert torch.equal(ta[key], tb[key]), key
    k = len(targets[0]["track_query_boxes"])
    assert k > 0
    torch.testing.assert_close(loss, ref_loss, rtol=1e-5, atol=1e-6)
    ref_flat = flat_of(step, ref)
    torch.testing.assert_close(step.flat_grad, ref_flat, rtol=2e-4, atol=1e-6 * float(ref_flat.abs().max()))


def test_softmax_entry_points_reject_bad_arguments():
    import ctypes
    from trackformer_b200 import _build, ext
    lib = ctypes.CDLL(_build.build_library())
    vp, i, f, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_int64
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, vp)
    cost = lib.tfb200_match_cost_softmax_f32
    cost.restype = i
    cost.argtypes = [vp] * 5 + [i64, i, i] + [f] * 3 + [vp]
    assert cost(None, p, p, p, p, 4, 21, 3, 1, 5, 2, None) == -1
    assert cost(p, p, p, p, p, 4, 1, 3, 1, 5, 2, None) == -2                       # no "no object" column
    assert cost(p, p, p, p, p, 0, 21, 3, 1, 5, 2, None) == 0                       # no rows: no-op
    track = lib.tfb200_match_cost_track_softmax_f32
    track.restype = i
    track.argtypes = [vp] * 6 + [i] * 5 + [f] * 3 + [vp]
    assert track(p, p, p, p, None, p, 1, 1, 4, 21, 3, 1, 5, 2, None) == -1         # NULL row_pin
    assert track(p, p, p, p, p, p, 1, 1, 4, 21, 1 << 20, 1, 5, 2, None) == -2      # T beyond shared memory
    loss = lib.tfb200_set_loss_fwd_softmax_f32
    loss.restype = i
    loss.argtypes = [vp] * 20 + [i] * 5 + [f, vp]
    args = [p] * 20
    assert loss(*args, 1, 1, 4, 21, 3, 0.0, None) == -2                            # eos_coef must be > 0
    no_norm = list(args)
    no_norm[15] = None
    assert loss(*no_norm, 1, 1, 4, 21, 3, 0.1, None) == -1                         # NULL row_norm
    bwd = lib.tfb200_set_loss_bwd_softmax_f32
    bwd.restype = i
    bwd.argtypes = [vp] * 10 + [i] * 4 + [vp]
    assert bwd(*([p] * 7), None, p, p, 1, 1, 4, 21, None) == -1                    # NULL ce_norm
    m = ext.load()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.match_cost_softmax(torch.zeros(4, 21), torch.zeros(4, 4), torch.zeros(3, dtype=torch.int64),
                             torch.zeros(3, 4), 1.0, 5.0, 2.0)
