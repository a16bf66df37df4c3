"""GPU parity tests of the MSDeformAttn hot path (run on an H100: ``pytest -m gpu``).

Every test goes through the product boundary -- the compiled module
``MultiScaleDeformableAttention`` / ``MSDeformAttnFunction`` (which call through the C ABI of
libmsda_b200.so) or the C ABI directly via ctypes -- and is checked against
  * the golden fixtures recorded from the reference's own function (tests/golden/), and
  * the oracle (plain-C restatement, oracle/msda_oracle.c) on seeded inputs, and
  * at full BASELINE sizes, size-independent properties (linearity, constant fields, adjointness).
Tolerances: fp32 1e-4 relative / 1e-4 absolute on O(1) data (summation order differs from the
reference's at::sum and the backward uses atomics); fp64 1e-10.  The reference's own tests
accept rtol 1e-2 / atol 1e-3 (ops/test.py:31).
"""
import ctypes

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden

pytestmark = pytest.mark.gpu

F32 = dict(rtol=1e-4, atol=1e-4)     # O(1) data, 16..64-term fp32 dot products with cancellation
F64 = dict(rtol=1e-10, atol=1e-12)


def assert_close_but_for_ties(actual, desired, rtol, atol, max_bad=4, err_msg=""):
    """assert_allclose that forgives a handful of elements.  grad_sampling_loc is DISCONTINUOUS where a sampling
    coordinate lands exactly on a pixel boundary: `loc * W - 0.5` is one fused multiply-add on the GPU (as in the
    reference's CUDA kernel, compiled with nvcc's default -fmad) but two roundings in the C oracle, so a sample that
    sits on the boundary to the last bit may take the other cell -- a different, equally valid one-sided derivative.
    With 11 M samples per full-size call that happens to about one element."""
    bad = ~np.isclose(actual, desired, rtol=rtol, atol=atol)
    if int(bad.sum()) > max_bad:
        np.testing.assert_allclose(actual, desired, rtol=rtol, atol=atol, err_msg=err_msg)


def tol(dt):
    return F32 if dt in (np.float32, torch.float32) else F64


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


@pytest.fixture(scope="module")
def msda(dev):
    from trackformer_b200 import ext
    return ext.load()


def to_dev(g, dev, keys=("value", "shapes", "loc", "attn", "grad_out")):
    return [torch.from_numpy(g[k]).to(dev) for k in keys]


# ----------------------------------------------------------------------------- golden fixtures
@pytest.mark.parametrize("name", golden_names())
def test_forward_matches_reference_fixture(msda, dev, name):
    g = load_golden(name)
    value, shapes, loc, attn, _ = to_dev(g, dev)
    out = msda.ms_deform_attn_forward(value, shapes, loc, attn, 64)
    np.testing.assert_allclose(out.cpu().numpy(), g["out"], **tol(g["value"].dtype))


@pytest.mark.parametrize("name", [n for n in golden_names() if n != "border_fwd_f64"])
def test_backward_matches_reference_fixture(msda, dev, name):
    g = load_golden(name)
    value, shapes, loc, attn, gout = to_dev(g, dev)
    gv, gl, ga = msda.ms_deform_attn_backward(value, shapes, loc, attn, gout, 64)
    t = tol(g["value"].dtype)
    np.testing.assert_allclose(gv.cpu().numpy(), g["grad_value"], **t)
    np.testing.assert_allclose(ga.cpu().numpy(), g["grad_attn"], **t)
    np.testing.assert_allclose(gl.cpu().numpy(), g["grad_loc"], rtol=t["rtol"] * 5, atol=t["atol"] * 50)


def test_reference_test_script_tolerances(dev):
    """ops/test.py:23-95 restated: autograd through MSDeformAttnFunction, loss = out.abs().sum(),
    allclose(rtol=1e-2, atol=1e-3) against the reference function's recorded results."""
    from trackformer_b200.msda_function import MSDeformAttnFunction
    for name in ("ref_test_f32", "ref_test_f64"):
        g = load_golden(name)
        value, shapes, loc, attn, _ = to_dev(g, dev)
        value.requires_grad_(True), loc.requires_grad_(True), attn.requires_grad_(True)
        out = MSDeformAttnFunction.apply(value, shapes, loc, attn, 2)
        assert torch.allclose(out.cpu(), torch.from_numpy(g["out"]), rtol=1e-2, atol=1e-3)
        gv, gl, ga = torch.autograd.grad(out.abs().sum(), (value, loc, attn))
        for got, key in ((gv, "grad_value"), (gl, "grad_loc"), (ga, "grad_attn")):
            assert torch.allclose(got.cpu(), torch.from_numpy(g[key]), rtol=1e-2, atol=1e-3), key


@pytest.mark.parametrize("which", ["value", "loc", "attn", "all"])
def test_gradcheck_fp64(dev, which):
    """ops/test_double_precision.py:98-119: gradcheck of the CUDA function in double precision."""
    from trackformer_b200.msda_function import MSDeformAttnFunction
    torch.manual_seed(3)
    N, M, D, Lq, L, P = 2, 2, 4, 3, 3, 2
    shapes = torch.as_tensor([(12, 8), (6, 4), (3, 2)], dtype=torch.long, device=dev)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    value = (torch.rand(N, S, M, D, dtype=torch.float64) * 0.01).to(dev)
    loc = torch.rand(N, Lq, M, L, P, 2, dtype=torch.float64).to(dev)
    attn = torch.rand(N, Lq, M, L, P, dtype=torch.float64).to(dev) + 1e-5
    attn = attn / attn.sum(-1, keepdim=True).sum(-2, keepdim=True)
    value.requires_grad_(which in ("value", "all"))
    loc.requires_grad_(which in ("loc", "all"))
    attn.requires_grad_(which in ("attn", "all"))
    assert torch.autograd.gradcheck(MSDeformAttnFunction.apply, (value, shapes, loc, attn, 2),
                                    nondet_tol=1e-12)


# ----------------------------------------------------------------------------- vs the C oracle
def rand_problem(seed, N, M, D, Lq, hw, P, dtype=np.float32, lo=-0.1, hi=1.1):
    rng = np.random.default_rng(seed)
    shapes = np.asarray(hw, dtype=np.int64)
    L = len(hw)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    value = rng.standard_normal((N, S, M, D)).astype(dtype)
    loc = rng.uniform(lo, hi, (N, Lq, M, L, P, 2)).astype(dtype)
    a = rng.standard_normal((N, Lq, M, L * P))
    a = np.exp(a - a.max(-1, keepdims=True))
    attn = (a / a.sum(-1, keepdims=True)).reshape(N, Lq, M, L, P).astype(dtype)
    gout = rng.standard_normal((N, Lq, M * D)).astype(dtype)
    return value, shapes, loc, attn, gout


ORACLE_CASES = {
    # name: (N, M, D, Lq, levels, P, dtype)
    "c1_decoder":   (1, 8, 32, 300, [(60, 80), (30, 40), (15, 20), (8, 10)], 4, np.float32),
    "c1_encoder":   (1, 8, 32, 6380, [(60, 80), (30, 40), (15, 20), (8, 10)], 4, np.float32),
    "batch2_d32":   (2, 8, 32, 517, [(25, 42), (13, 21), (7, 11), (4, 6)], 4, np.float32),
    "d36_l8":       (1, 8, 36, 311, [(17, 30), (9, 15), (5, 8), (3, 4)] * 2, 4, np.float32),
    "d36_heads3_thin": (2, 3, 36, 50, [(1, 7), (6, 1), (2, 2), (5, 9)], 2, np.float32),      # nine-lane kernel, M != 8
    "d36_l4_batch2": (2, 8, 36, 1001, [(34, 60), (17, 30), (9, 15), (5, 8)], 4, np.float32),
    "d64_heads4":   (1, 4, 64, 129, [(9, 11), (5, 6)], 4, np.float32),
    "d16":          (2, 8, 16, 65, [(9, 11), (5, 6)], 4, np.float32),
    "d8_p3":        (1, 3, 8, 77, [(7, 9), (4, 5), (2, 3)], 3, np.float32),
    "d5_scalar":    (2, 3, 5, 33, [(6, 7), (3, 4)], 2, np.float32),
    "d3_f64":       (1, 2, 3, 19, [(4, 5)], 5, np.float64),
    "d32_f64":      (1, 8, 32, 101, [(12, 16), (6, 8), (3, 4), (2, 2)], 4, np.float64),
    "d100_wide":    (1, 2, 100, 21, [(4, 5), (2, 3)], 2, np.float32),
    "single_pixel": (1, 1, 4, 5, [(1, 1)], 1, np.float32),
}


@pytest.mark.parametrize("name", sorted(ORACLE_CASES))
def test_forward_backward_match_c_oracle(msda, dev, name):
    from oracle import msda_oracle
    N, M, D, Lq, hw, P, dt = ORACLE_CASES[name]
    value, shapes, loc, attn, gout = rand_problem(hash(name) % 1000, N, M, D, Lq, hw, P, dt)
    ref_out = msda_oracle.msda_forward(value, shapes, loc, attn)
    ref_gv, ref_gl, ref_ga = msda_oracle.msda_backward(value, shapes, loc, attn, gout)
    tv, ts, tl, ta, tg = (torch.from_numpy(x).to(dev) for x in (value, shapes, loc, attn, gout))
    out = msda.ms_deform_attn_forward(tv, ts, tl, ta, 64)
    gv, gl, ga = msda.ms_deform_attn_backward(tv, ts, tl, ta, tg, 64)
    t = tol(dt)
    np.testing.assert_allclose(out.cpu().numpy(), ref_out, **t)
    # grad_value cells on coarse levels accumulate thousands of terms -> scale atol with magnitude
    scale = max(1.0, float(np.abs(ref_gv).max()))
    np.testing.assert_allclose(gv.cpu().numpy(), ref_gv, rtol=t["rtol"], atol=t["atol"] * scale)
    np.testing.assert_allclose(ga.cpu().numpy(), ref_ga, **t)
    np.testing.assert_allclose(gl.cpu().numpy(), ref_gl, rtol=t["rtol"] * 5, atol=t["atol"] * 50)


def test_d36_forward_kernel_equals_generic_kernel(msda, dev):
    """the nine-lane D = 36 forward (msda_d36.cuh) against the generic kernel (variant 1) on the same inputs"""
    value, shapes, loc, attn, _ = rand_problem(36, 2, 8, 36, 777, [(20, 33), (10, 17), (5, 9), (3, 5)] * 2, 4, np.float32)
    tv, ts, tl, ta = (torch.from_numpy(x).to(dev) for x in (value, shapes, loc, attn))
    fast = msda.ms_deform_attn_forward(tv, ts, tl, ta, 64)
    msda.set_variant(1, 0)
    try:
        generic = msda.ms_deform_attn_forward(tv, ts, tl, ta, 64)
    finally:
        msda.set_variant(0, 0)
    torch.testing.assert_close(fast, generic, rtol=1e-5, atol=1e-6)


def test_unaligned_views_take_the_scalar_path(msda, dev):
    """value / grad_output views whose data pointer is not 16-byte aligned must still be exact."""
    from oracle import msda_oracle
    value, shapes, loc, attn, gout = rand_problem(5, 1, 2, 4, 23, [(5, 6), (3, 3)], 2)
    S = value.shape[1]
    big = torch.zeros(value.size + 1, device=dev)
    v_un = big[1:].view(1, S, 2, 4)
    v_un.copy_(torch.from_numpy(value))
    assert v_un.data_ptr() % 16 != 0 and v_un.is_contiguous()
    ts, tl, ta, tg = (torch.from_numpy(x).to(dev) for x in (shapes, loc, attn, gout))
    out = msda.ms_deform_attn_forward(v_un, ts, tl, ta, 64)
    np.testing.assert_allclose(out.cpu().numpy(), msda_oracle.msda_forward(value, shapes, loc, attn), **F32)
    gv, gl, ga = msda.ms_deform_attn_backward(v_un, ts, tl, ta, tg, 64)
    rgv, rgl, rga = msda_oracle.msda_backward(value, shapes, loc, attn, gout)
    np.testing.assert_allclose(gv.cpu().numpy(), rgv, **F32)
    np.testing.assert_allclose(ga.cpu().numpy(), rga, **F32)


# ----------------------------------------------------------------------------- C ABI via ctypes
@pytest.fixture(scope="module")
def cabi(dev):
    from trackformer_b200 import ext
    lib = ctypes.CDLL(ext.library_path())
    vp, i = ctypes.c_void_p, ctypes.c_int
    lib.msda_b200_forward_f32.argtypes = [vp] * 5 + [i] * 7 + [vp]
    lib.msda_b200_backward_f32.argtypes = [vp] * 8 + [i] * 7 + [vp]
    lib.msda_b200_forward_host_f32.argtypes = [vp] * 5 + [i] * 7 + [i]
    lib.msda_b200_backward_host_f32.argtypes = [vp] * 8 + [i] * 7 + [i]
    lib.msda_b200_launch_count.restype = ctypes.c_uint64
    return lib


def test_c_abi_device_pointers(cabi, dev):
    from oracle import msda_oracle
    N, M, D, Lq, hw, P = 2, 8, 32, 211, [(20, 27), (10, 14), (5, 7), (3, 4)], 4
    value, shapes, loc, attn, gout = rand_problem(21, N, M, D, Lq, hw, P)
    S, L = value.shape[1], len(hw)
    tv, ts, tl, ta, tg = (torch.from_numpy(x).to(dev) for x in (value, shapes, loc, attn, gout))
    out = torch.empty(N, Lq, M * D, device=dev)
    gv, gl, ga = torch.full_like(tv, 7.0), torch.empty_like(tl), torch.empty_like(ta)   # gv is zero-filled by the callee
    stream = torch.cuda.current_stream(dev).cuda_stream
    before = cabi.msda_b200_launch_count()
    rc = cabi.msda_b200_forward_f32(tv.data_ptr(), ts.data_ptr(), tl.data_ptr(), ta.data_ptr(), out.data_ptr(),
                                    N, S, M, D, L, Lq, P, stream)
    assert rc == 0
    rc = cabi.msda_b200_backward_f32(tv.data_ptr(), ts.data_ptr(), tl.data_ptr(), ta.data_ptr(), tg.data_ptr(),
                                     gv.data_ptr(), gl.data_ptr(), ga.data_ptr(), N, S, M, D, L, Lq, P, stream)
    assert rc == 0
    torch.cuda.synchronize(dev)
    assert cabi.msda_b200_launch_count() == before + 2
    np.testing.assert_allclose(out.cpu().numpy(), msda_oracle.msda_forward(value, shapes, loc, attn), **F32)
    rgv, rgl, rga = msda_oracle.msda_backward(value, shapes, loc, attn, gout)
    np.testing.assert_allclose(gv.cpu().numpy(), rgv, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(ga.cpu().numpy(), rga, **F32)
    np.testing.assert_allclose(gl.cpu().numpy(), rgl, rtol=5e-4, atol=5e-4)


def test_c_abi_host_buffers(cabi, dev):
    from oracle import msda_oracle
    N, M, D, Lq, hw, P = 1, 8, 32, 97, [(12, 16), (6, 8), (3, 4), (2, 2)], 4
    value, shapes, loc, attn, gout = rand_problem(22, N, M, D, Lq, hw, P)
    S, L = value.shape[1], len(hw)
    out = np.empty((N, Lq, M * D), np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert cabi.msda_b200_forward_host_f32(p(value), p(shapes), p(loc), p(attn), p(out), N, S, M, D, L, Lq, P, 0) == 0
    np.testing.assert_allclose(out, msda_oracle.msda_forward(value, shapes, loc, attn), **F32)
    gv, gl, ga = np.empty_like(value), np.empty_like(loc), np.empty_like(attn)
    assert cabi.msda_b200_backward_host_f32(p(value), p(shapes), p(loc), p(attn), p(gout), p(gv), p(gl), p(ga),
                                            N, S, M, D, L, Lq, P, 0) == 0
    rgv, rgl, rga = msda_oracle.msda_backward(value, shapes, loc, attn, gout)
    np.testing.assert_allclose(gv, rgv, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(ga, rga, **F32)
    np.testing.assert_allclose(gl, rgl, rtol=5e-4, atol=5e-4)


# ----------------------------------------------------------------------------- error behaviour
def test_error_behaviour(msda, dev):
    value = torch.zeros(2, 4, 1, 4, device=dev)
    shapes = torch.tensor([[2, 2]], device=dev)
    loc = torch.zeros(2, 1, 1, 1, 1, 2, device=dev)
    attn = torch.zeros(2, 1, 1, 1, 1, device=dev)
    with pytest.raises(RuntimeError, match="contiguous"):               # ms_deform_attn_cuda.cu:29
        nc = torch.zeros(2, 4, 4, 2, device=dev).transpose(2, 3)          # [2,4,2,4], not contiguous
        msda.ms_deform_attn_forward(nc, shapes, torch.zeros(2, 1, 2, 1, 1, 2, device=dev),
                                    torch.zeros(2, 1, 2, 1, 1, device=dev), 64)
    with pytest.raises(RuntimeError, match="CUDA tensor"):              # ms_deform_attn_cuda.cu:32
        msda.ms_deform_attn_forward(value, shapes.cpu(), loc, attn, 64)
    with pytest.raises(RuntimeError, match="must divide"):              # ms_deform_attn_cuda.cu:48
        msda.ms_deform_attn_forward(torch.zeros(3, 4, 1, 4, device=dev), shapes,
                                    torch.zeros(3, 1, 1, 1, 1, 2, device=dev), torch.zeros(3, 1, 1, 1, 1, device=dev), 2)
    with pytest.raises(RuntimeError, match="float32 or float64"):
        msda.ms_deform_attn_forward(value.half(), shapes, loc.half(), attn.half(), 64)
    out = msda.ms_deform_attn_forward(value, shapes, loc, attn, 64)      # N=2, step=min(2,64)=2: fine
    assert out.shape == (2, 1, 4)


def test_empty_query_set(msda, dev):
    value = torch.randn(1, 4, 2, 4, device=dev)
    shapes = torch.tensor([[2, 2]], device=dev)
    out = msda.ms_deform_attn_forward(value, shapes, torch.zeros(1, 0, 2, 1, 1, 2, device=dev),
                                      torch.zeros(1, 0, 2, 1, 1, device=dev), 64)
    assert out.shape == (1, 0, 8)
    gv, gl, ga = msda.ms_deform_attn_backward(value, shapes, torch.zeros(1, 0, 2, 1, 1, 2, device=dev),
                                              torch.zeros(1, 0, 2, 1, 1, device=dev),
                                              torch.zeros(1, 0, 8, device=dev), 64)
    assert not gv.any() and gl.numel() == 0 and ga.numel() == 0


# ----------------------------------------------------------------------------- full-size properties
C2_LEVELS = [(100, 167), (50, 84), (25, 42), (13, 21)]       # 1x3x800x1333, SURVEY section 8
C5_LEVELS = [(135, 240), (68, 120), (34, 60), (17, 30)]      # 1x3x1080x1920


def gpu_problem(dev, seed, N, M, D, Lq, hw, P, lo=0.0, hi=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    shapes = torch.as_tensor(hw, dtype=torch.long)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    L = len(hw)
    value = torch.randn(N, S, M, D, generator=g).to(dev)
    loc = (torch.rand(N, Lq, M, L, P, 2, generator=g) * (hi - lo) + lo).to(dev)
    attn = torch.softmax(torch.randn(N, Lq, M, L * P, generator=g), -1).view(N, Lq, M, L, P).to(dev)
    return value, shapes.to(dev), loc, attn


@pytest.mark.parametrize("cfg", ["c2_encoder", "c5_encoder_d36", "c5_decoder_l8"])
def test_full_size_properties(msda, dev, cfg):
    if cfg == "c2_encoder":
        N, M, D, hw, P = 1, 8, 32, C2_LEVELS, 4
        Lq = sum(h * w for h, w in hw)
    elif cfg == "c5_encoder_d36":
        N, M, D, hw, P = 1, 8, 36, C5_LEVELS, 4
        Lq = sum(h * w for h, w in hw)
    else:
        N, M, D, hw, P, Lq = 1, 8, 36, C5_LEVELS * 2, 4, 800
    value, shapes, loc, attn = gpu_problem(dev, 7, N, M, D, Lq, hw, P, -0.05, 1.05)
    f = lambda v, a: msda.ms_deform_attn_forward(v, shapes, loc, a, 64)
    out = f(value, attn)
    assert torch.isfinite(out).all()
    # (1) linearity in value and in the attention weights
    v2 = torch.randn_like(value)
    torch.testing.assert_close(f(2 * value - 3 * v2, attn), 2 * out - 3 * f(v2, attn), rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(f(value, 0.25 * attn), 0.25 * out, rtol=1e-5, atol=1e-6)
    # (2) constant field + strictly interior samples: out = const * sum(attn) = const
    loc_in = loc.clamp(0.06, 0.94)      # > 0.5/min(H,W): all four corners of every sample inside
    ones = torch.full_like(value, 1.5)
    out_c = msda.ms_deform_attn_forward(ones, shapes, loc_in, attn, 64)
    torch.testing.assert_close(out_c, torch.full_like(out_c, 1.5), rtol=1e-5, atol=1e-5)
    # (3) adjointness: <out, g> == <value, grad_value>,  grad_attn . attn == <out, g>
    gout = torch.randn_like(out)
    gv, gl, ga = msda.ms_deform_attn_backward(value, shapes, loc, attn, gout, 64)
    lhs = (out.double() * gout.double()).sum()
    torch.testing.assert_close((value.double() * gv.double()).sum(), lhs, rtol=1e-4, atol=1e-2)
    torch.testing.assert_close((attn.double() * ga.double()).sum(), lhs, rtol=1e-4, atol=1e-2)
    # (4) total mass: with an all-ones grad_output and interior samples every bilinear tap spreads
    #     weight 1 -> sum(grad_value) == D * sum(attn) == D * N * Lq * M
    gv1, _, _ = msda.ms_deform_attn_backward(value, shapes, loc_in, attn, torch.ones_like(out), 64)
    torch.testing.assert_close(gv1.double().sum(), torch.tensor(float(D * N * Lq * M), dtype=torch.float64, device=dev),
                               rtol=1e-4, atol=1.0)
    # (5) finite-difference check of grad_loc on a few coordinates.  One location element only moves one
    #     (q, m) output row; bilinear interpolation is piecewise linear, so the central difference is exact
    #     unless the +-eps probe crosses a pixel border (skipped) -- what remains is fp32 rounding.
    L = len(hw)
    eps = 2e-5
    checked = 0
    gen = torch.Generator().manual_seed(1)
    flat_gl = gl.reshape(-1)
    for i in torch.randint(0, loc.numel(), (24,), generator=gen).tolist():
        c = i % 2
        p_ = (i // 2) % P
        l_ = (i // (2 * P)) % L
        m_ = (i // (2 * P * L)) % M
        q_ = (i // (2 * P * L * M)) % Lq
        size = hw[l_][1] if c == 0 else hw[l_][0]
        t = float(loc.reshape(-1)[i]) * size - 0.5
        import math
        if not (0.0 < t < size - 1.0) or math.floor(t - 2 * eps * size) != math.floor(t + 2 * eps * size):
            continue
        lp, lm = loc.clone().reshape(-1), loc.clone().reshape(-1)
        lp[i] += eps
        lm[i] -= eps
        op = msda.ms_deform_attn_forward(value, shapes, lp.view_as(loc), attn, 64)[0, q_, m_ * D:(m_ + 1) * D]
        om = msda.ms_deform_attn_forward(value, shapes, lm.view_as(loc), attn, 64)[0, q_, m_ * D:(m_ + 1) * D]
        g_row = gout[0, q_, m_ * D:(m_ + 1) * D].double()
        fd = float(((op.double() - om.double()) * g_row).sum() / (float(lp[i]) - float(lm[i])))
        got = float(flat_gl[i])
        assert abs(fd - got) <= 0.03 * (abs(fd) + abs(got)) + 0.5, (i, fd, got)
        checked += 1
    assert checked >= 8


def test_backward_determinism_of_loc_and_attn_grads(msda, dev):
    value, shapes, loc, attn = gpu_problem(dev, 9, 1, 8, 32, 300, C2_LEVELS, 4)
    gout = torch.randn(1, 300, 256, device=dev)
    a = msda.ms_deform_attn_backward(value, shapes, loc, attn, gout, 64)
    b = msda.ms_deform_attn_backward(value, shapes, loc, attn, gout, 64)
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])       # no atomics on these two
    torch.testing.assert_close(a[0], b[0], rtol=1e-5, atol=1e-5)     # grad_value: atomic order may differ


# ----------------------------------------------------------------------------- tiled encoder forward
TILE_CASES = {
    "c1_enc": (1, 8, [(60, 80), (30, 40), (15, 20), (8, 10)], 4, "model"),
    "c2_enc_n2": (2, 8, [(100, 167), (50, 84), (25, 42), (13, 21)], 4, "model"),
    "odd_sizes": (1, 8, [(37, 53), (19, 27), (10, 14), (5, 7)], 4, "model"),
    "wide_offsets": (1, 8, [(40, 56), (20, 28), (10, 14), (5, 7)], 4, "uniform"),       # boxes overflow -> global path
    "two_levels_p8": (1, 8, [(24, 40), (12, 20)], 8, "model"),
    "heads4": (1, 4, [(33, 47), (17, 24), (9, 12)], 4, "model"),
    "smooth_c1": (2, 8, [(60, 80), (30, 40), (15, 20), (8, 10)], 4, "smooth"),
    "l8_p4": (1, 8, [(20, 30), (10, 15), (5, 8), (3, 4)] * 2, 4, "model"),
}


@pytest.mark.parametrize("name", sorted(TILE_CASES))
def test_tiled_encoder_forward_equals_general_kernel(msda, dev, name):
    """The shared-memory tiled kernel against the default kernel (same taps) and against the oracle."""
    from oracle import msda_oracle
    N, M, hw, P, dist = TILE_CASES[name]
    g = torch.Generator().manual_seed(len(name))
    shapes = torch.as_tensor(hw, dtype=torch.long)
    L = len(hw)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    value = torch.randn(N, S, M, 32, generator=g)
    if dist == "uniform":
        loc = torch.rand(N, S, M, L, P, 2, generator=g) * 1.2 - 0.1
    else:
        refs = []
        for (h, w) in hw:
            ys, xs = torch.meshgrid(torch.arange(h) + 0.5, torch.arange(w) + 0.5, indexing="ij")
            refs.append(torch.stack([xs.reshape(-1) / w, ys.reshape(-1) / h], -1))
        ref = torch.cat(refs, 0)[None, :, None, None, None, :]
        if dist == "smooth":         # what a model produces: per-(head, level, point) offsets + a little jitter
            off = torch.randn(1, 1, M, L, P, 2, generator=g) * 2.5 + 0.2 * torch.randn(N, S, M, L, P, 2, generator=g)
        else:
            off = torch.randn(N, S, M, L, P, 2, generator=g) * 2.5
        loc = ref + off / shapes.flip(-1).float()[None, None, None, :, None, :]
    attn = torch.softmax(torch.randn(N, S, M, L * P, generator=g), -1).view(N, S, M, L, P)
    tv, ts, tl, ta = value.to(dev), shapes.to(dev), loc.to(dev), attn.to(dev)
    flat_hw = [int(v) for pair in hw for v in pair]
    if P == 4 and L <= 4:            # the tiled kernel's domain: make sure IT produced the numbers, not the fallback
        tiled = msda.ms_deform_attn_forward_enc_strict(tv, ts, tl, ta, flat_hw, 64)
    else:
        with pytest.raises(RuntimeError):
            msda.ms_deform_attn_forward_enc_strict(tv, ts, tl, ta, flat_hw, 64)
        tiled = msda.ms_deform_attn_forward_enc(tv, ts, tl, ta, flat_hw, 64)
    general = msda.ms_deform_attn_forward(tv, ts, tl, ta, 64)
    torch.testing.assert_close(tiled, general, rtol=1e-5, atol=1e-5)     # different summation order, same taps
    ref_out = msda_oracle.msda_forward(value.numpy(), shapes.numpy(), loc.numpy(), attn.numpy())
    np.testing.assert_allclose(tiled.cpu().numpy(), ref_out, **F32)


@pytest.mark.parametrize("name", sorted(TILE_CASES))
def test_tiled_encoder_backward_matches_c_oracle(msda, dev, name):
    """The TMA-staged backward tile kernel (strict: no fallback inside its domain) against the C restatement of the
    reference's backward kernels, on the same encoder-shaped problems as the kernel families below."""
    from oracle import msda_oracle
    N, M, hw, P, dist = TILE_CASES[name]
    value, shapes, loc, attn, gout = _encoder_problem(name)
    ref_gv, ref_gl, ref_ga = msda_oracle.msda_backward(value.numpy(), shapes.numpy(), loc.numpy(), attn.numpy(), gout.numpy())
    tv, ts, tl, ta, tg = (x.to(dev) for x in (value, shapes, loc, attn, gout))
    flat_hw = [int(v) for pair in hw for v in pair]
    if P == 4 and len(hw) <= 4:
        gv, gl, ga = msda.ms_deform_attn_backward_enc_strict(tv, ts, tl, ta, tg, flat_hw, 64)
    else:
        with pytest.raises(RuntimeError):
            msda.ms_deform_attn_backward_enc_strict(tv, ts, tl, ta, tg, flat_hw, 64)
        gv, gl, ga = msda.ms_deform_attn_backward_enc(tv, ts, tl, ta, tg, flat_hw, 64)
    torch.cuda.synchronize()
    scale = max(1.0, float(np.abs(ref_gv).max()))
    np.testing.assert_allclose(gv.cpu().numpy(), ref_gv, rtol=F32["rtol"], atol=F32["atol"] * scale)
    np.testing.assert_allclose(ga.cpu().numpy(), ref_ga, **F32)
    assert_close_but_for_ties(gl.cpu().numpy(), ref_gl, rtol=F32["rtol"] * 5, atol=F32["atol"] * 50)


# ----------------------------------------------------------------------------- every fp32 / D = 32 kernel family
def _encoder_problem(name, D=32):
    N, M, hw, P, dist = TILE_CASES[name]
    g = torch.Generator().manual_seed(100 + len(name))
    shapes = torch.as_tensor(hw, dtype=torch.long)
    L = len(hw)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    value = torch.randn(N, S, M, D, generator=g)
    if dist == "uniform":
        loc = torch.rand(N, S, M, L, P, 2, generator=g) * 1.2 - 0.1
    else:
        refs = []
        for (h, w) in hw:
            ys, xs = torch.meshgrid(torch.arange(h) + 0.5, torch.arange(w) + 0.5, indexing="ij")
            refs.append(torch.stack([xs.reshape(-1) / w, ys.reshape(-1) / h], -1))
        ref = torch.cat(refs, 0)[None, :, None, None, None, :]
        # smooth offsets (what a model produces: neighbouring queries sample neighbouring windows, so the run
        # kernels take their "same window" / "slide by one" paths) plus a little per-sample jitter
        base = torch.randn(1, 1, M, L, P, 2, generator=g) * 2.5
        off = base + 0.2 * torch.randn(N, S, M, L, P, 2, generator=g)
        loc = ref + off / shapes.flip(-1).float()[None, None, None, :, None, :]
    attn = torch.softmax(torch.randn(N, S, M, L * P, generator=g), -1).view(N, S, M, L, P)
    attn[:, ::7, 1] = 0.0                                     # exact-zero attention rows (skipped reductions)
    gout = torch.randn(N, S, M * D, generator=g)
    return value, shapes, loc, attn, gout


# 0 = automatic choice, 100 / 101 = run kernels (R = 8 / 4), 120 / 121 = second-generation run kernels (4 / 2 slots
# interleaved), 110 = warp-per-group kernels, 20 = 8-lane-group kernels
@pytest.mark.parametrize("variant", [0, 100, 101, 110, 120, 121, 20])
@pytest.mark.parametrize("name", sorted(TILE_CASES))
def test_kernel_families_match_c_oracle(msda, dev, name, variant):
    """Forward and fused backward of every specialised kernel family on encoder-shaped problems (incl. the FULL
    C2 encoder call, batch 2) against the C restatement of the reference kernels."""
    from oracle import msda_oracle
    value, shapes, loc, attn, gout = _encoder_problem(name)
    ref_out = msda_oracle.msda_forward(value.numpy(), shapes.numpy(), loc.numpy(), attn.numpy())
    ref_gv, ref_gl, ref_ga = msda_oracle.msda_backward(value.numpy(), shapes.numpy(), loc.numpy(), attn.numpy(),
                                                       gout.numpy())
    tv, ts, tl, ta, tg = (x.to(dev) for x in (value, shapes, loc, attn, gout))
    msda.set_variant(variant, variant)
    try:
        out = msda.ms_deform_attn_forward(tv, ts, tl, ta, 64)
        gv, gl, ga = msda.ms_deform_attn_backward(tv, ts, tl, ta, tg, 64)
        torch.cuda.synchronize()
    finally:
        msda.set_variant(0, 0)
    np.testing.assert_allclose(out.cpu().numpy(), ref_out, **F32)
    scale = max(1.0, float(np.abs(ref_gv).max()))
    np.testing.assert_allclose(gv.cpu().numpy(), ref_gv, rtol=F32["rtol"], atol=F32["atol"] * scale)
    np.testing.assert_allclose(ga.cpu().numpy(), ref_ga, **F32)
    assert_close_but_for_ties(gl.cpu().numpy(), ref_gl, rtol=F32["rtol"] * 5, atol=F32["atol"] * 50)


@pytest.mark.parametrize("variant", [100, 101, 110, 120, 121])
def test_kernel_families_on_degenerate_and_ragged_shapes(msda, dev, variant):
    """levels with a single row / column (on-the-fly predicated path), Lq not a multiple of the run block, M = 4 and
    12 heads, L*P = 64 (the largest supported; > 48 KB of dynamic shared memory), out-of-range locations"""
    from oracle import msda_oracle
    cases = [(2, 8, 77, [(1, 7), (6, 1), (2, 2), (5, 9)], 2), (1, 4, 1000, [(9, 11), (5, 6)], 4),
             (1, 12, 301, [(12, 16), (6, 8), (3, 4)], 3), (1, 8, 190, [(6, 8), (3, 4)] * 4, 8)]
    for i, (N, M, Lq, hw, P) in enumerate(cases):
        value, shapes, loc, attn, gout = rand_problem(50 + i, N, M, 32, Lq, hw, P, np.float32, lo=-0.3, hi=1.3)
        ref_out = msda_oracle.msda_forward(value, shapes, loc, attn)
        ref_gv, ref_gl, ref_ga = msda_oracle.msda_backward(value, shapes, loc, attn, gout)
        tv, ts, tl, ta, tg = (torch.from_numpy(x).to(dev) for x in (value, shapes, loc, attn, gout))
        msda.set_variant(variant, variant)
        try:
            out = msda.ms_deform_attn_forward(tv, ts, tl, ta, 64)
            gv, gl, ga = msda.ms_deform_attn_backward(tv, ts, tl, ta, tg, 64)
            torch.cuda.synchronize()
        finally:
            msda.set_variant(0, 0)
        np.testing.assert_allclose(out.cpu().numpy(), ref_out, **F32, err_msg=str(i))
        scale = max(1.0, float(np.abs(ref_gv).max()))
        np.testing.assert_allclose(gv.cpu().numpy(), ref_gv, rtol=F32["rtol"], atol=F32["atol"] * scale, err_msg=str(i))
        np.testing.assert_allclose(ga.cpu().numpy(), ref_ga, **F32, err_msg=str(i))
        np.testing.assert_allclose(gl.cpu().numpy(), ref_gl, rtol=F32["rtol"] * 5, atol=F32["atol"] * 50, err_msg=str(i))


def test_d32_kernels_with_64_samples_per_query(msda, dev):
    """ADVICE r1: the 8-lane-group backward needs > 48 KB of dynamic shared memory once L*P >= 38"""
    from oracle import msda_oracle
    value, shapes, loc, attn, gout = rand_problem(64, 1, 8, 32, 130, [(6, 8), (3, 4)] * 4, 8, np.float32)
    ref_gv, ref_gl, ref_ga = msda_oracle.msda_backward(value, shapes, loc, attn, gout)
    tv, ts, tl, ta, tg = (torch.from_numpy(x).to(dev) for x in (value, shapes, loc, attn, gout))
    msda.set_variant(20, 20)
    try:
        gv, gl, ga = msda.ms_deform_attn_backward(tv, ts, tl, ta, tg, 64)
        torch.cuda.synchronize()
    finally:
        msda.set_variant(0, 0)
    np.testing.assert_allclose(ga.cpu().numpy(), ref_ga, **F32)
    np.testing.assert_allclose(gv.cpu().numpy(), ref_gv, rtol=F32["rtol"], atol=F32["atol"] * max(1.0, float(np.abs(ref_gv).max())))


@pytest.mark.parametrize("variant", [0, 100, 101])
@pytest.mark.parametrize("name", ["c1_enc", "odd_sizes", "wide_offsets", "heads4", "l8_p4"])
def test_run_kernels_d36_match_c_oracle(msda, dev, name, variant):
    """the published TrackFormer geometry (hidden 288, D = 36: nine lanes per head row, three runs per warp), forward
    and fused backward of the run kernels against the C oracle"""
    from oracle import msda_oracle
    value, shapes, loc, attn, gout = _encoder_problem(name, D=36)
    ref_out = msda_oracle.msda_forward(value.numpy(), shapes.numpy(), loc.numpy(), attn.numpy())
    ref_gv, ref_gl, ref_ga = msda_oracle.msda_backward(value.numpy(), shapes.numpy(), loc.numpy(), attn.numpy(),
                                                       gout.numpy())
    tv, ts, tl, ta, tg = (x.to(dev) for x in (value, shapes, loc, attn, gout))
    msda.set_variant(variant, variant)
    try:
        out = msda.ms_deform_attn_forward(tv, ts, tl, ta, 64)
        gv, gl, ga = msda.ms_deform_attn_backward(tv, ts, tl, ta, tg, 64)
        torch.cuda.synchronize()
    finally:
        msda.set_variant(0, 0)
    np.testing.assert_allclose(out.cpu().numpy(), ref_out, **F32)
    scale = max(1.0, float(np.abs(ref_gv).max()))
    np.testing.assert_allclose(gv.cpu().numpy(), ref_gv, rtol=F32["rtol"], atol=F32["atol"] * scale)
    np.testing.assert_allclose(ga.cpu().numpy(), ref_ga, **F32)
    np.testing.assert_allclose(gl.cpu().numpy(), ref_gl, rtol=F32["rtol"] * 5, atol=F32["atol"] * 50)


@pytest.mark.parametrize("D", [32, 36])
def test_fused_prologue_equals_module_chain(msda, dev, D):
    """MSDeformAttnFusedFunction (softmax + location arithmetic in the kernel prologue, SURVEY 8(f1)) against the
    materialising chain softmax -> locations -> MSDeformAttnFunction on the same projection, forward and both gradients"""
    from trackformer_b200.msda_function import MSDeformAttnFunction, MSDeformAttnFusedFunction
    hw = [(37, 53), (19, 27), (10, 14), (5, 7)]
    g = torch.Generator().manual_seed(D)
    shapes = torch.as_tensor(hw, dtype=torch.long)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    N, M, L, P = 2, 8, 4, 4
    value = torch.randn(N, S, M, D, generator=g).to(dev).requires_grad_(True)
    proj = torch.randn(N, S, 3 * M * L * P, generator=g)
    proj[..., :2 * M * L * P] *= 2.0
    proj = proj.to(dev).requires_grad_(True)
    refs = []
    for (h, w) in hw:
        ys, xs = torch.meshgrid(torch.arange(h) + 0.5, torch.arange(w) + 0.5, indexing="ij")
        refs.append(torch.stack([xs.reshape(-1) / w, ys.reshape(-1) / h], -1))
    ref = torch.cat(refs, 0)[None, :, None, :].expand(N, S, L, 2).contiguous().to(dev)
    gout = torch.randn(N, S, M * D, generator=g).to(dev)
    ts = shapes.to(dev)

    out = MSDeformAttnFusedFunction.apply(value, ts, proj, ref, P)
    out.backward(gout)
    gv, gp = value.grad.clone(), proj.grad.clone()
    value.grad = proj.grad = None

    n_off = 2 * M * L * P
    offsets = proj[..., :n_off].reshape(N, S, M, L, P, 2)
    attn = torch.softmax(proj[..., n_off:].reshape(N, S, M, L * P), -1).view(N, S, M, L, P)
    loc = ref[:, :, None, :, None, :] + offsets / ts.float()[None, None, None, :, None, :]      # (H, W) as stored
    exp = MSDeformAttnFunction.apply(value, ts, loc, attn, 64)
    exp.backward(gout)
    torch.testing.assert_close(out, exp, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(gv, value.grad, rtol=1e-4, atol=1e-4 * float(value.grad.abs().max()))
    torch.testing.assert_close(gp, proj.grad, rtol=2e-3, atol=2e-4 * float(proj.grad.abs().max()))


@pytest.mark.parametrize("spread", [0.6, 6.0])
@pytest.mark.parametrize("hw", [[(37, 53), (19, 27), (10, 14), (5, 7)], [(60, 80), (30, 40), (15, 20), (8, 10)]])
def test_fused_prologue_tile_kernels_equal_module_chain(msda, dev, hw, spread):
    """MSDeformAttnEncFusedFunction (TMA tile kernels with softmax + location arithmetic in the tap pass) against the
    materialising chain on the same projection: forward, grad_value and the projection gradient (offsets and logits through
    the softmax).  spread = 6 px pushes many samples out of the staged boxes (per-sample path) and out of the image."""
    from trackformer_b200.msda_function import MSDeformAttnEncFusedFunction, MSDeformAttnFunction
    g = torch.Generator().manual_seed(int(spread * 10) + hw[0][0])
    shapes = torch.as_tensor(hw, dtype=torch.long)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    N, M, L, P, D = 2, 8, 4, 4, 32
    value = torch.randn(N, S, M, D, generator=g).to(dev).requires_grad_(True)
    proj = torch.randn(N, S, 3 * M * L * P, generator=g)
    proj[..., :2 * M * L * P] *= spread
    proj = proj.to(dev).requires_grad_(True)
    refs = []
    for (h, w) in hw:
        ys, xs = torch.meshgrid(torch.arange(h) + 0.5, torch.arange(w) + 0.5, indexing="ij")
        refs.append(torch.stack([xs.reshape(-1) / w, ys.reshape(-1) / h], -1))
    ref = torch.cat(refs, 0)[None, :, None, :].expand(N, S, L, 2).contiguous().to(dev)
    gout = torch.randn(N, S, M * D, generator=g).to(dev)
    ts = shapes.to(dev)
    flat_hw = [int(v) for pair in hw for v in pair]

    out = MSDeformAttnEncFusedFunction.apply(value, proj, ref, flat_hw)
    out.backward(gout)
    gv, gp = value.grad.clone(), proj.grad.clone()
    value.grad = proj.grad = None

    n_off = 2 * M * L * P
    offsets = proj[..., :n_off].reshape(N, S, M, L, P, 2)
    attn = torch.softmax(proj[..., n_off:].reshape(N, S, M, L * P), -1).view(N, S, M, L, P)
    loc = ref[:, :, None, :, None, :] + offsets / ts.float()[None, None, None, :, None, :]      # (H, W) as stored
    exp = MSDeformAttnFunction.apply(value, ts, loc, attn, 64)
    exp.backward(gout)
    torch.testing.assert_close(out, exp, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(gv, value.grad, rtol=1e-4, atol=1e-4 * float(value.grad.abs().max()))
    bad = ~torch.isclose(gp, proj.grad, rtol=2e-3, atol=2e-4 * float(proj.grad.abs().max()))
    assert int(bad.sum()) <= 4, int(bad.sum())                # (ties on pixel boundaries, see assert_close_but_for_ties)
