"""The encoder FFN with its activation fused into the wgmma TF32 GEMM (csrc/tf32_gemm.cu, relu_dropout / dropout_grad
epilogues; fused_linear.ffn) against fp64 products and the hash restatement of tests/dropout_hash.py.

Tolerance as in test_tf32_gemm_gpu.py: TF32 operands, fp32 accumulation -> 2e-3 of the result scale.  The keep mask is
compared exactly wherever the pre-activation is clear of TF32 rounding (its sign is then the same in every product
order)."""
import pytest
import torch

import dropout_hash as dh

pytestmark = pytest.mark.gpu

KEEP = 0.9
SHAPES = [  # (M tokens, K in-features, N out-features); M % 128 != 0 everywhere: a ragged last row tile
    (22223, 256, 1024), (44446, 256, 1024), (5000, 256, 1024), (22223, 1024, 256), (5000, 1024, 256),
]


@pytest.fixture(scope="module")
def op(cuda_device):
    from trackformer_b200 import ext
    return ext.load()


@pytest.fixture
def tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _data(dev, M, K, N, seed=0):
    g = torch.Generator().manual_seed(seed + M + K + N)
    x = torch.randn(M, K, generator=g).to(dev)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
    b = (0.1 * torch.randn(N, generator=g)).to(dev)
    return x, w, b


def _rel(a, ref):
    return float((a.detach().double() - ref).abs().max() / ref.abs().max())


def _seed(s, dev):
    return torch.tensor([s], dtype=torch.int64, device=dev)


@pytest.mark.parametrize("M,K,N", SHAPES)
def test_relu_dropout_epilogue(op, cuda_device, M, K, N):
    x, w, b = _data(cuda_device, M, K, N)
    a = x.double() @ w.double().t() + b.double()
    seed = 0x1234_5678_9ABC + M
    h = op.tf32_linear_relu_dropout(x, w, b, _seed(seed, cuda_device), KEEP, True)
    mask = dh.relu_dropout_mask(seed, (M, N), KEEP, cuda_device)
    clear = a.abs() > 4e-3 * float(a.abs().max())
    assert torch.equal((h > 0)[clear], (mask & (a > 0))[clear])
    assert _rel(h, torch.where(mask & (a > 0), a / KEEP, torch.zeros_like(a))) < 2e-3
    # the unfused kernel on the same pre-activation keeps the same elements
    h_unfused = op.relu_dropout_forward(op.tf32_linear(x, w, b, False), _seed(seed, cuda_device), KEEP, True)
    assert torch.equal((h > 0)[clear], (h_unfused > 0)[clear])
    # eval: plain ReLU, no seed
    assert _rel(op.tf32_linear_relu_dropout(x, w, b, None, KEEP, False), a.clamp_min(0)) < 2e-3
    h3 = op.tf32_linear_relu_dropout(x.view(1, M, K), w, b, None, KEEP, False)
    assert h3.shape == (1, M, N)


@pytest.mark.parametrize("M,K,N", SHAPES)
def test_dropout_grad_epilogue(op, cuda_device, M, K, N):
    """ga = h > 0 ? (dy . w) / keep : 0 for dy [M, N], w [N, K], h [M, K] -- relu_dropout_backward on the product"""
    x, w, _ = _data(cuda_device, M, K, N, seed=1)
    g = torch.Generator().manual_seed(M)
    dy = torch.randn(M, N, generator=g).to(cuda_device)
    h = op.relu_dropout_forward(x, _seed(99 + M, cuda_device), KEEP, True)        # any relu_dropout output [M, K]
    prod = dy.double() @ w.double()
    ref = torch.where(h > 0, prod / KEEP, torch.zeros_like(prod))
    ga = op.tf32_linear_dgrad_relu_dropout(dy, w, h, KEEP, True)
    assert ga.shape == (M, K)
    assert _rel(ga, ref) < 2e-3
    unfused = op.relu_dropout_backward(op.tf32_linear_dgrad(dy, w), h, KEEP, True)
    assert _rel(ga, unfused.double()) < 2e-3
    # eval: the ReLU mask only
    ref_eval = torch.where(h > 0, prod, torch.zeros_like(prod))
    assert _rel(op.tf32_linear_dgrad_relu_dropout(dy, w, h, KEEP, False), ref_eval) < 2e-3


@pytest.mark.parametrize("M", [22223, 5000])
def test_ffn_autograd_matches_fp64(op, cuda_device, tf32, monkeypatch, M):
    """fused_linear.ffn: output and the gradients of x, w1, b1, w2, b2 against an fp64 restatement with the mask the
    kernel drew.  The mask is read off the kernel's h > 0 (test_relu_dropout_epilogue pins it to the hash): where the
    pre-activation is within rounding of zero, an fp64 sign can differ, and in the backward one such element would move a
    whole gradient entry."""
    from trackformer_b200 import fused_linear as fl
    torch.manual_seed(0)
    l1, l2 = torch.nn.Linear(256, 1024).to(cuda_device), torch.nn.Linear(1024, 256).to(cuda_device)
    drop = torch.nn.Dropout(1 - KEEP)
    g = torch.Generator().manual_seed(M)
    x = torch.randn(1, M, 256, generator=g).to(cuda_device).requires_grad_(True)
    gy = torch.randn(1, M, 256, generator=g).to(cuda_device)
    assert fl.ffn_fusable(x, l1, l2, drop)
    seed = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=cuda_device)
    monkeypatch.setattr(fl.seeds, "next_seed", lambda device: seed)
    y = fl.ffn(x, l1, l2, drop)
    y.backward(gy)
    grads = [x.grad, l1.weight.grad, l1.bias.grad, l2.weight.grad, l2.bias.grad]

    xs = [t.detach().double().requires_grad_(True) for t in (x, l1.weight, l1.bias, l2.weight, l2.bias)]
    a = xs[0] @ xs[1].t() + xs[2]
    mask = op.tf32_linear_relu_dropout(x.detach(), l1.weight.detach(), l1.bias.detach(), seed, KEEP, True) > 0
    hr = torch.where(mask, a / KEEP, torch.zeros_like(a))
    yr = hr @ xs[3].t() + xs[4]
    yr.backward(gy.double())
    assert _rel(y, yr.detach()) < 2e-3
    for got, r in zip(grads, xs):
        assert got.shape == r.shape
        assert _rel(got, r.grad) < 2e-3


def test_composition_runs_under_strict_fp32_and_short_token_axes(cuda_device, monkeypatch):
    """the fused route is TF32-only and long-token-only: elsewhere forward_ffn calls relu_dropout as before"""
    from trackformer_b200 import deformable_transformer as dt
    from trackformer_b200 import fused_linear as fl
    layer = dt.DeformableTransformerEncoderLayer(256, 1024, 0.1).to(cuda_device).train()
    calls = []
    monkeypatch.setattr(dt, "relu_dropout", lambda a, d: calls.append(a.shape) or fl.relu_dropout(a, d))
    monkeypatch.setattr(fl, "_TCGEN05", True)
    old = torch.backends.cuda.matmul.allow_tf32
    try:
        for tf32, rows, fused in ((False, 5000, False), (True, 2047, False), (True, 5000, True)):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            calls.clear()
            src = torch.randn(1, rows, 256, device=cuda_device, requires_grad=True)
            layer.forward_ffn(src).sum().backward()
            assert calls == ([] if fused else [(1, rows, 1024)]), (tf32, rows)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def test_graph_replays_draw_different_masks(op, cuda_device):
    """the seed is read on the device: a captured call draws a fresh mask on every replay"""
    M, K, N = 4097, 256, 1024
    x, w, b = _data(cuda_device, M, K, N, seed=3)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for _ in range(2):                           # warm-up outside the capture
            op.tf32_linear_relu_dropout(x, w, b, _seed(1, cuda_device), KEEP, True)
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        seed = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=cuda_device)
        h = op.tf32_linear_relu_dropout(x, w, b, seed, KEEP, True)
    a = x.double() @ w.double().t() + b.double()
    clear = a.abs() > 4e-3 * float(a.abs().max())
    kept = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        mask = dh.relu_dropout_mask(int(seed.item()), (M, N), KEEP, cuda_device) & (a > 0)
        assert torch.equal((h > 0)[clear], mask[clear])
        kept.append(h > 0)
    assert not torch.equal(kept[0], kept[1])
