"""The hand-written wgmma TF32 Linear (csrc/tf32_gemm.cu): forward (+bias, +ReLU), dgrad (MN-major weight operand),
split-token wgrad (TMA reduce-add) against fp64 products.  Tolerance: TF32 operands (10-bit mantissa, truncated by the
tensor core) with fp32 accumulation -> ~1e-3 of the result scale, the same class as cuBLAS' TF32 kernels, whose error
is printed next to ours."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [  # (M tokens, K in-features, N out-features)
    (22223, 256, 256), (22223, 256, 384), (4097, 256, 1024), (4097, 1024, 256), (300, 256, 256), (127, 128, 128),
    (1, 128, 128), (129, 256, 128),
]


@pytest.fixture(scope="module")
def op(cuda_device):
    from trackformer_b200 import ext
    return ext.load()


def _data(dev, M, K, N, seed=0):
    g = torch.Generator().manual_seed(seed + M + K + N)
    x = torch.randn(M, K, generator=g).to(dev)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    gy = torch.randn(M, N, generator=g).to(dev)
    return x, w, b, gy


def _rel(a, ref):
    return float((a.double() - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("M,K,N", SHAPES)
def test_forward_bias_relu(op, cuda_device, M, K, N):
    assert op.tf32_linear_supported(M, N, K)
    x, w, b, _ = _data(cuda_device, M, K, N)
    ref = x.double() @ w.double().t() + b.double()
    assert _rel(op.tf32_linear(x, w, b, False), ref) < 2e-3
    assert _rel(op.tf32_linear(x, w, b, True), ref.clamp_min(0)) < 2e-3
    assert _rel(op.tf32_linear(x, w, None, False), x.double() @ w.double().t()) < 2e-3
    y3 = op.tf32_linear(x.view(1, M, K), w, b, False)                 # leading dimensions are kept
    assert y3.shape == (1, M, N)


@pytest.mark.parametrize("M,K,N", SHAPES)
def test_dgrad_and_wgrad(op, cuda_device, M, K, N):
    x, w, _, gy = _data(cuda_device, M, K, N, seed=1)
    assert _rel(op.tf32_linear_dgrad(gy, w), gy.double() @ w.double()) < 2e-3
    dw_ref = gy.double().t() @ x.double()
    dw = op.tf32_linear_wgrad(gy, x)
    assert dw.shape == (N, K)
    assert _rel(dw, dw_ref) < 2e-3
    torch.testing.assert_close(op.tf32_linear_wgrad(gy, x), dw, rtol=1e-5, atol=1e-5 * float(dw_ref.abs().max()))  # re-zeroed


def test_unsupported_shapes_are_refused(op, cuda_device):
    assert not op.tf32_linear_supported(100, 100, 256) and not op.tf32_linear_supported(100, 128, 100)
    x = torch.zeros(64, 100, device=cuda_device)
    with pytest.raises(RuntimeError):
        op.tf32_linear(x, torch.zeros(128, 100, device=cuda_device), None, False)


def test_fused_linear_autograd_matches_library(cuda_device, monkeypatch):
    """trackformer_b200.fused_linear.linear with the wgmma path on: outputs and all three gradients against F.linear"""
    import trackformer_b200.fused_linear as fl
    monkeypatch.setattr(fl, "_TCGEN05", True)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        x, w, b, gy = _data(cuda_device, 5000, 256, 384, seed=2)
        xs = [t.clone().requires_grad_(True) for t in (x, w, b)]
        y = fl.linear(xs[0].view(1, 5000, 256), xs[1], xs[2])
        y.backward(gy.view(1, 5000, 384))
        rs = [t.double().clone().requires_grad_(True) for t in (x, w, b)]
        yr = torch.nn.functional.linear(rs[0], rs[1], rs[2])
        yr.backward(gy.double())
        assert _rel(y.view(5000, 384), yr.detach()) < 2e-3
        for a, r in zip(xs, rs):
            assert _rel(a.grad, r.grad) < 2e-3
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
