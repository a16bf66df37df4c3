"""Every route of ``MSDeformAttn.forward`` pinned to an fp64 restatement of the reference, with the route forced.

The module picks one of several kernel chains per call (trackformer_b200/msda_module.py), and in the default ``auto``
mode three encoder decisions are made by timing both candidates on the first call, so a model-level test only sees the
route that won on its machine.  Here each route is forced (tests/msda_module_reference.py ``forced_route``), the
bindings it called are asserted, and the output and every gradient -- query, ``input_flatten``, ``reference_points``
where it requires grad, and all eight parameter gradients -- are compared with fp64 autograd through the reference's
own arithmetic (ops/modules/ms_deform_attn.py:60-89):

====  ==========================================================  =============================================
route how it is reached                                           bindings
====  ==========================================================  =============================================
E1    encoder, D = 32, L = P = 4, fused tile chosen               ``*_enc_fused`` (TMA tile kernels, softmax and
                                                                  locations in the tap pass)
E2-5  encoder, fused tile not chosen; tile or direct forward      ``sampling_prep_*`` + ``*_enc`` (tile, proven
      and backward                                                by the ``*_strict`` bindings) or general kernels
E6    ``TFB200_FUSED_PREP=1``, L * P = 16, Lq >= 2048             ``ms_deform_attn_{forward,backward}_fused``
E7/D3 ``query_attn_mask`` given, or reference points with grad    torch softmax / locations + core
D1/D2 decoder, 4-d or 2-d references without grad                 ``sampling_prep_*`` + general kernels
MF    multi-frame: hidden 288 (D = 36), 8 levels                  ``*_enc`` refused by the tile kernels, general
                                                                  run kernels
====  ==========================================================  =============================================

Gradients are compared on the rows without a sample within fp32 rounding (1e-4 px on a 240 px side) of a bilinear cell
boundary (the upstream gradient of the others is zeroed on both sides; see ``kinked``); the forward on every row.  Bounds
are elementwise against max|reference| of each tensor, plus a relative L2 bound, with no looser group for any parameter.
The padded batch of two (distinct reference points per image and per level) is what pins the tile kernels' per-level
reference read; a dense batch of one has the same normalised reference on every level.
"""
import math

import pytest
import torch

import msda_module_reference as mref

pytestmark = pytest.mark.gpu

C2 = [(100, 167), (50, 84), (25, 42), (13, 21)]          # 800 x 1333 at strides 8..64
C5 = [(135, 240), (68, 120), (34, 60), (17, 30)]         # 1080 x 1920
ODD = [(37, 53), (19, 27), (10, 14), (5, 7)]             # tile tails in both axes on every level
TINY = [(8, 12), (4, 6), (2, 3), (1, 2)]                 # coarsest level one pixel tall: outside the tile kernels' domain
GEOMS = {"c2": (C2, 2), "c5": (C5, 1), "odd": (ODD, 2), "tiny": (TINY, 2)}

OUT_BOUND, INPUT_BOUND, PARAM_BOUND, REL_L2 = 2e-5, 5e-5, 1e-4, 1e-5
MAX_KINKED = 0.10

_PREP = {"sampling_prep_forward", "sampling_prep_backward"}
ROUTES = {
    "E1_fused_tile": (dict(tiled_enc_fused="1"),
                      {"ms_deform_attn_forward_enc_fused", "ms_deform_attn_backward_enc_fused"}),
    "E2_tile_tile": (dict(tiled_enc="1", tiled_enc_bwd="1"),
                     _PREP | {"ms_deform_attn_forward_enc", "ms_deform_attn_backward_enc"}),
    "E3_tile_direct": (dict(tiled_enc="1"), _PREP | {"ms_deform_attn_forward_enc", "ms_deform_attn_backward"}),
    "E4_direct_tile": (dict(tiled_enc_bwd="1"), _PREP | {"ms_deform_attn_forward", "ms_deform_attn_backward_enc"}),
    "E5_direct_direct": (dict(), _PREP | {"ms_deform_attn_forward", "ms_deform_attn_backward"}),
    "E6_fused_prep": (dict(fused_prep=True), {"ms_deform_attn_forward_fused", "ms_deform_attn_backward_fused"}),
}


@pytest.fixture(scope="module", autouse=True)
def _free_cache_at_teardown():
    yield
    _CACHE.clear()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


@pytest.fixture()
def strict_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# ------------------------------------------------------------------------------------------------------------------
# problems
# ------------------------------------------------------------------------------------------------------------------
def _shapes(hw, device):
    t = torch.tensor(hw, dtype=torch.long, device=device)
    t._hw_list = list(hw)
    return t


def _level_padding(hw, batch, device):
    """[N, S] padding of a batch whose second image covers ~80 % x 70 % of every level, and the valid ratios [N, L, 2]
    (w, h).  A batch of one is dense."""
    masks, ratios = [], []
    for h, w in hw:
        m = torch.zeros(batch, h, w, dtype=torch.bool)
        r = [[1.0, 1.0]] * batch
        if batch > 1:
            vh, vw = math.ceil(0.8 * h), math.ceil(0.7 * w)
            m[1, vh:] = True
            m[1, :, vw:] = True
            r[1] = [vw / w, vh / h]
        masks.append(m.flatten(1))
        ratios.append(torch.tensor(r))
    pad = torch.cat(masks, 1).to(device) if batch > 1 else None
    return pad, torch.stack(ratios, 1).to(device)


def _module(d_model, levels, weights, seed, device):
    """MSDeformAttn at the reference initialisation ("init"), moved off it ("perturbed": every parameter + N(0, 0.02),
    offsets within a pixel or so) or with wide offsets ("far": offset weights N(0, 0.375), ~6 px per unit query)."""
    from trackformer_b200.msda_module import MSDeformAttn
    torch.manual_seed(seed)
    mod = MSDeformAttn(d_model, levels, 8, 4)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        if weights in ("perturbed", "far"):
            for p in mod.parameters():
                p.add_(torch.randn(p.shape, generator=g) * 0.02)
        if weights == "far":
            mod.sampling_offsets.weight.copy_(torch.randn(mod.sampling_offsets.weight.shape, generator=g) * 6.0
                                              / math.sqrt(d_model))
    return mod.to(device)


class _Problem:
    """Module, fp32 inputs, the fp64 reference (output, gradients) and the kinked-row mask of one geometry."""

    def __init__(self, mod, query, ref, x, hw, pad, attn_mask, gout, grad_inputs, with_grad):
        self.mod, self.query, self.ref, self.x, self.hw, self.pad, self.attn_mask = mod, query, ref, x, hw, pad, attn_mask
        self.shapes = _shapes(hw, query.device)
        self.with_grad = with_grad
        self.inputs = {"query": query, "input_flatten": x, "reference_points": ref}
        self.grad_inputs = grad_inputs
        P = mref.params64(mod)
        q64, ref64, x64 = (t.detach().double() for t in (query, ref, x))
        with torch.no_grad():
            loc = mref.sampling_locations64(P, q64, ref64, hw, n_levels=mod.n_levels)
        self.kinked = mref.kinked(loc, hw)
        del loc
        leaves = {"query": q64, "input_flatten": x64, "reference_points": ref64}
        for k in grad_inputs:
            leaves[k].requires_grad_(True)
        out = mref.msda_fp64(P, leaves["query"], leaves["reference_points"], leaves["input_flatten"], hw, pad, attn_mask,
                             n_levels=mod.n_levels)
        self.out = out.detach()
        self.grads = {}
        if with_grad:
            self.gout = gout * ~self.kinked[..., None]
            out.backward(self.gout.double())
            self.grads = {k: leaves[k].grad for k in grad_inputs}
            self.grads.update({k: v.grad for k, v in P.items()})
        del out, P, leaves


_CACHE = {}


def _cached(key, build):
    """One problem at a time (the routes of one geometry run back to back and share the fp64 reference)."""
    if key not in _CACHE:
        _CACHE.clear()
        torch.cuda.empty_cache()
        _CACHE[key] = build()
    return _CACHE[key]


def _encoder_problem(geom, weights, with_grad=True, attn_mask=False, d_model=256, hw=None, batch=None, seed=0):
    def build():
        dev = torch.device("cuda:0")
        lvl_hw, n = (hw, batch) if hw is not None else GEOMS[geom]
        from trackformer_b200.deformable_transformer import DeformableTransformerEncoder
        s = sum(h * w for h, w in lvl_hw)
        pad, ratios = _level_padding(lvl_hw, n, dev)
        ref = DeformableTransformerEncoder.get_reference_points(_shapes(lvl_hw, dev), ratios, dev)
        g = torch.Generator().manual_seed(seed + 7)
        query = torch.randn(n, s, d_model, generator=g).to(dev)
        x = torch.randn(n, s, d_model, generator=g).to(dev)
        gout = torch.randn(n, s, d_model, generator=g).to(dev)
        mask = None
        if attn_mask:
            mask = torch.zeros(n, s, dtype=torch.bool)
            mask[:, ::7] = True
            mask = mask.to(dev)
        mod = _module(d_model, len(lvl_hw), weights, seed, dev)
        return _Problem(mod, query, ref, x, lvl_hw, pad, mask, gout, ("query", "input_flatten"), with_grad)
    return _cached(("enc", geom, weights, with_grad, attn_mask, d_model, str(hw), batch, seed), build)


def _decoder_problem(kind, ref_grad, attn_mask, d_model=256, hw=C2, batch=2, queries=300, tracks=40, seed=1):
    def build():
        dev = torch.device("cuda:0")
        s, lq = sum(h * w for h, w in hw), tracks + queries
        pad, ratios = _level_padding(hw, batch, dev)
        g = torch.Generator().manual_seed(seed + 11)
        query = torch.randn(batch, lq, d_model, generator=g).to(dev)
        x = torch.randn(batch, s, d_model, generator=g).to(dev)
        gout = torch.randn(batch, lq, d_model, generator=g).to(dev)
        boxes = torch.cat([torch.rand(batch, lq, 2, generator=g) * 0.6 + 0.2,
                           torch.rand(batch, lq, 2, generator=g) * 0.25 + 0.05], -1).to(dev)
        if kind == 4:
            ref = boxes[:, :, None] * torch.cat([ratios, ratios], -1)[:, None]
        else:
            ref = boxes[:, :, None, :2] * ratios[:, None]
        ref = ref.contiguous()
        mask = None
        if attn_mask:                                       # filler track slots at the tail of each image's 40
            mask = torch.zeros(batch, lq, dtype=torch.bool)
            mask[0, 31:tracks] = True
            mask[-1, 17:tracks] = True
            mask = mask.to(dev)
        mod = _module(d_model, len(hw), "perturbed", seed, dev)
        grads = ("query", "input_flatten") + (("reference_points",) if ref_grad else ())
        return _Problem(mod, query, ref, x, hw, pad, mask, gout, grads, True)
    return _cached(("dec", kind, ref_grad, attn_mask, d_model, str(hw), batch, queries, tracks, seed), build)


# ------------------------------------------------------------------------------------------------------------------
# running a route and comparing
# ------------------------------------------------------------------------------------------------------------------
def _run(pb, switches):
    """Forward (and backward of the kink-masked upstream gradient) of the module on fresh leaves, under the forced
    route.  Returns (output, {name: grad}, spy)."""
    leaves = {k: v.detach().clone().requires_grad_(k in pb.grad_inputs and pb.with_grad) for k, v in pb.inputs.items()}
    pb.mod.zero_grad(set_to_none=True)
    with mref.forced_route(**switches) as spy:
        with torch.set_grad_enabled(pb.with_grad):
            out = pb.mod(leaves["query"], leaves["reference_points"], leaves["input_flatten"], pb.shapes, pb.pad,
                         pb.attn_mask)
            if pb.with_grad:
                out.backward(pb.gout)
        torch.cuda.synchronize()
        grads = {}
        if pb.with_grad:
            grads = {k: leaves[k].grad for k in pb.grad_inputs}
            grads.update({k: p.grad for k, p in pb.mod.named_parameters()})
    return out.detach(), grads, spy


def _compare(pb, out, grads, tag):
    kinked = float(pb.kinked.double().mean())
    assert kinked < MAX_KINKED, f"{tag}: {kinked:.1%} of the rows have a sample on a cell boundary"
    rows = []

    def one(name, got, want, bound):
        got, want = got.double(), want.double()
        scale = float(want.abs().max())
        assert scale > 0, f"{tag}: reference {name} is all zeros"
        err = float((got - want).abs().max()) / scale
        rel = float(torch.linalg.vector_norm(got - want) / torch.linalg.vector_norm(want))
        rows.append((name, err, bound, rel))

    one("output", out, pb.out, OUT_BOUND)
    for name, want in pb.grads.items():
        one(f"grad {name}", grads[name], want, INPUT_BOUND if name in pb.inputs else PARAM_BOUND)
    report = "\n".join(f"  {n:34s} max {e:.2e} (bound {b:.0e})  rel L2 {r:.2e}" for n, e, b, r in rows)
    print(f"\n[{tag}] kinked rows {kinked:.2%}\n{report}")
    bad = [n for n, e, b, r in rows if not (e <= b and r <= REL_L2)]
    assert not bad, f"{tag}: {bad} out of bounds (kinked rows {kinked:.2%})\n{report}"


def _expect(spy, names, with_grad=True):
    want = set(names) if with_grad else {n for n in names if "backward" not in n}
    assert spy.names == want, f"bindings {sorted(spy.names)}, expected {sorted(want)}"
    if any(n.endswith("_enc") for n in want):
        spy.prove_tiles()


# ------------------------------------------------------------------------------------------------------------------
# encoder routes E1-E6 at C2 (batch 2, padded), C5 and odd sizes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("geom", ["c2", "c5", "odd"])
def test_encoder_route_matches_fp64(cuda_device, strict_fp32, geom, route):
    pb = _encoder_problem(geom, "perturbed")
    switches, names = ROUTES[route]
    out, grads, spy = _run(pb, switches)
    _expect(spy, names)
    _compare(pb, out, grads, f"{route} {geom}")


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("geom", ["c2", "odd"])
def test_encoder_route_far_offsets_match_fp64(cuda_device, strict_fp32, geom, route):
    """~6 px offsets: samples leave the staged boxes of the tile kernels and the image."""
    pb = _encoder_problem(geom, "far")
    switches, names = ROUTES[route]
    out, grads, spy = _run(pb, switches)
    _expect(spy, names)
    _compare(pb, out, grads, f"{route} {geom} far")


@pytest.mark.parametrize("route", list(ROUTES))
def test_encoder_route_forward_at_reference_init_matches_fp64(cuda_device, strict_fp32, route):
    """The compass-grid offsets of the reference initialisation put the samples on pixel centres (nearly every row is
    kinked, so only the forward is compared)."""
    pb = _encoder_problem("c2", "init", with_grad=False)
    switches, names = ROUTES[route]
    out, _, spy = _run(pb, switches)
    _expect(spy, names, with_grad=False)
    err = float((out.double() - pb.out).abs().max()) / float(pb.out.abs().max())
    rel = float(torch.linalg.vector_norm(out.double() - pb.out) / torch.linalg.vector_norm(pb.out))
    assert err <= OUT_BOUND and rel <= REL_L2, (err, rel)


@pytest.mark.parametrize("core", ["tile", "direct"])
@pytest.mark.parametrize("geom", ["c2", "odd"])
def test_encoder_query_attn_mask_route_matches_fp64(cuda_device, strict_fp32, geom, core):
    """E7: a query_attn_mask sends the encoder call through the torch softmax / locations into the encoder core."""
    pb = _encoder_problem(geom, "perturbed", attn_mask=True)
    if core == "tile":
        switches, names = dict(tiled_enc="1", tiled_enc_bwd="1"), {"ms_deform_attn_forward_enc",
                                                                   "ms_deform_attn_backward_enc"}
    else:
        switches, names = dict(), {"ms_deform_attn_forward", "ms_deform_attn_backward"}
    out, grads, spy = _run(pb, switches)
    _expect(spy, names)
    _compare(pb, out, grads, f"E7 {core} {geom}")


# ------------------------------------------------------------------------------------------------------------------
# a one-pixel coarsest level: outside the tile kernels' domain
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["auto", "fused_forced"])
def test_encoder_with_one_pixel_level_takes_unfused_route_and_matches_fp64(cuda_device, strict_fp32, mode):
    """A padded image side of 64 px or less makes the stride-64 level one pixel tall.  The fused tile route must not be
    taken there (its bindings raise outside the domain), neither when timed nor when forced."""
    pb = _encoder_problem("tiny", "perturbed")
    switches = (dict(tiled_enc="auto", tiled_enc_bwd="auto", tiled_enc_fused="auto") if mode == "auto"
                else dict(tiled_enc_fused="1"))
    out, grads, spy = _run(pb, switches)
    assert not any("enc_fused" in n for n in spy.names), sorted(spy.names)
    assert spy.tiles_refused() == spy.names & {"ms_deform_attn_forward_enc", "ms_deform_attn_backward_enc"}
    _compare(pb, out, grads, f"tiny {mode}")


# ------------------------------------------------------------------------------------------------------------------
# decoder routes D1-D3 and the query_attn_mask route
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("attn_mask", [False, True], ids=["no_mask", "query_attn_mask"])
@pytest.mark.parametrize("ref_grad", [False, True], ids=["ref_detached", "ref_grad"])
@pytest.mark.parametrize("kind", [4, 2], ids=["boxes", "points"])
def test_decoder_route_matches_fp64(cuda_device, strict_fp32, kind, ref_grad, attn_mask):
    """300 object queries after 40 track slots into C2 memory of a padded batch of two."""
    pb = _decoder_problem(kind, ref_grad, attn_mask)
    core = {"ms_deform_attn_forward", "ms_deform_attn_backward"}
    out, grads, spy = _run(pb, {})
    _expect(spy, core if (ref_grad or attn_mask) else core | _PREP)
    _compare(pb, out, grads, f"decoder {kind}-d ref_grad={ref_grad} mask={attn_mask}")


# ------------------------------------------------------------------------------------------------------------------
# multi-frame: hidden 288 (D = 36), 8 levels (two frames of four)
# ------------------------------------------------------------------------------------------------------------------
MF_HW = [(50, 84), (25, 42), (13, 21), (7, 11)] * 2         # two 400 x 667 frames


def test_multi_frame_encoder_matches_fp64(cuda_device, strict_fp32):
    """Outside the tile kernels (D = 36, eight levels): with the tile kernels asked for, the extension serves the call
    with the general kernels (the R = 4 run kernels at this size), and says so through the strict bindings."""
    pb = _encoder_problem("mf", "perturbed", d_model=288, hw=MF_HW, batch=2)
    out, grads, spy = _run(pb, dict(tiled_enc="1", tiled_enc_bwd="1", tiled_enc_fused="1"))
    assert spy.names == _PREP | {"ms_deform_attn_forward_enc", "ms_deform_attn_backward_enc"}, sorted(spy.names)
    assert spy.tiles_refused() == {"ms_deform_attn_forward_enc", "ms_deform_attn_backward_enc"}
    _compare(pb, out, grads, "multi-frame encoder")


def test_multi_frame_decoder_matches_fp64(cuda_device, strict_fp32):
    """500 object queries after 30 track slots, 4-d references, into the two-frame memory."""
    pb = _decoder_problem(4, False, False, d_model=288, hw=MF_HW, batch=2, queries=500, tracks=30)
    out, grads, spy = _run(pb, {})
    _expect(spy, _PREP | {"ms_deform_attn_forward", "ms_deform_attn_backward"})
    _compare(pb, out, grads, "multi-frame decoder")


# ------------------------------------------------------------------------------------------------------------------
# the fused tile route's domain predicate against the bindings
# ------------------------------------------------------------------------------------------------------------------
DOMAIN_GEOMS = {
    "one_pixel_tall": ([(8, 12), (4, 6), (2, 3), (1, 2)], 8),
    "one_pixel_wide": ([(8, 12), (4, 6), (3, 2), (2, 1)], 8),
    "one_pixel": ([(8, 12), (4, 6), (2, 3), (1, 1)], 8),
    "level_of_two": ([(8, 12), (4, 6), (2, 3), (2, 2)], 8),
    "odd": (ODD, 8),
    "side_4095": ([(4095, 2), (2, 2), (2, 2), (2, 2)], 8),
    "side_4096_forward_only": ([(4096, 2), (2, 2), (2, 2), (2, 2)], 8),
    "s_2_20_forward_only": ([(1024, 1024), (2, 2), (2, 2), (2, 2)], 1),
    "s_below_2_20": ([(1023, 1024), (4, 4), (2, 2), (2, 2)], 1),
}


@pytest.mark.parametrize("name", list(DOMAIN_GEOMS))
def test_fused_tile_domain_predicate_matches_bindings(cuda_device, name):
    """``enc_fused_domain`` is true exactly when the fused tile bindings (and the strict tile bindings) accept the
    geometry, forward and backward, so that the module's gate and the kernels' check cannot drift apart."""
    from trackformer_b200 import ext
    from trackformer_b200.msda_function import enc_fused_domain
    msda = ext.load()
    hw, m = DOMAIN_GEOMS[name]
    dev = cuda_device
    flat = [v for pair in hw for v in pair]
    n, s, d = 1, sum(h * w for h, w in hw), 32
    value = torch.randn(n, s, m, d, device=dev)
    proj = torch.zeros(n, s, 3 * m * 16, device=dev)
    ref = torch.full((n, s, 4, 2), 0.5, device=dev)
    gout = torch.randn(n, s, m * d, device=dev)
    shapes = torch.tensor(hw, dtype=torch.long, device=dev)
    loc = torch.full((n, s, m, 4, 4, 2), 0.5, device=dev)
    attn = torch.full((n, s, m, 4, 4), 1.0 / 16, device=dev)

    def accepts(fn, *args):
        try:
            fn(*args)
        except RuntimeError as e:
            assert "not supported" in str(e) or "outside the tiled kernel's domain" in str(e), str(e)
            return False
        torch.cuda.synchronize()
        return True

    for backward in (False, True):
        want = enc_fused_domain(flat, n, s, m, d, s, backward=backward)
        if backward:
            got = {"enc_fused": accepts(msda.ms_deform_attn_backward_enc_fused, value, proj, ref, gout, flat),
                   "strict": accepts(msda.ms_deform_attn_backward_enc_strict, value, shapes, loc, attn, gout, flat, 64)}
        else:
            got = {"enc_fused": accepts(msda.ms_deform_attn_forward_enc_fused, value, proj, ref, flat),
                   "strict": accepts(msda.ms_deform_attn_forward_enc_strict, value, shapes, loc, attn, flat, 64)}
        assert got == {"enc_fused": want, "strict": want}, (name, "backward" if backward else "forward", want, got)
    expected = {"side_4096_forward_only": (True, False), "s_2_20_forward_only": (True, False)}.get(
        name, (name in ("level_of_two", "odd", "side_4095", "s_below_2_20"),) * 2)
    assert (enc_fused_domain(flat, n, s, m, d, s, backward=False),
            enc_fused_domain(flat, n, s, m, d, s, backward=True)) == expected
