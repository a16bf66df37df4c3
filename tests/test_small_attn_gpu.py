"""The decoder's query self-attention on the hand-written small-attention kernels (csrc/small_attn.cu) against PyTorch:
the attention core (forward, all three gradients, key-padding mask, strided [L, B, H, 32] views), the dropout path
(deterministic for a given seed: gradients checked against finite differences of the SAME masked function), and the
whole nn.MultiheadAttention replacement against the stock module with identical parameters."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def op(cuda_device):
    from trackformer_b200 import ext
    return ext.load()


def _ref(q, k, v, key_pad, scale):
    # q, k, v: [L, B, H, 32] -> [B, H, L, 32]
    qq, kk, vv = (t.permute(1, 2, 0, 3).double() for t in (q, k, v))
    s = qq @ kk.transpose(-1, -2) * scale
    if key_pad is not None:
        s = s.masked_fill(key_pad[:, None, None, :], float("-inf"))
    return (torch.softmax(s, -1) @ vv).permute(2, 0, 1, 3)


@pytest.mark.parametrize("L,B,H,masked", [(300, 1, 8, False), (77, 2, 8, True), (800, 1, 8, True), (33, 3, 4, False)])
def test_core_matches_pytorch(op, cuda_device, L, B, H, masked):
    from trackformer_b200.small_attention import _SmallAttention
    g = torch.Generator().manual_seed(L + B)
    packed = torch.randn(L, B, 3 * H * 32, generator=g).to(cuda_device)          # strided views of a packed projection
    q, k, v = (packed[..., i * H * 32:(i + 1) * H * 32].unflatten(-1, (H, 32)).detach().requires_grad_(True) for i in range(3))
    key_pad = None
    if masked:
        key_pad = torch.zeros(B, L, dtype=torch.bool, device=cuda_device)
        key_pad[:, L - 9:] = True
        key_pad[0, 3] = True
    scale = 32 ** -0.5
    out = _SmallAttention.apply(q, k, v, key_pad, None, scale, 1.0)
    gout = torch.randn(L, B, H, 32, generator=g).to(cuda_device)
    out.backward(gout)
    qr, kr, vr = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = _ref(qr, kr, vr, key_pad, scale)
    ref.backward(gout.double())
    torch.testing.assert_close(out.double(), ref, rtol=1e-4, atol=1e-5)
    for a, r in ((q, qr), (k, kr), (v, vr)):
        torch.testing.assert_close(a.grad.double(), r.grad, rtol=1e-4, atol=2e-5)


def test_dropout_is_deterministic_and_differentiated_consistently(op, cuda_device):
    from trackformer_b200.small_attention import _SmallAttention
    g = torch.Generator().manual_seed(5)
    L, B, H = 64, 1, 2
    q, k, v = (torch.randn(L, B, H, 32, generator=g).to(cuda_device).requires_grad_(True) for _ in range(3))
    seed = torch.tensor([1234567], dtype=torch.int64, device=cuda_device)
    w = torch.randn(L, B, H, 32, generator=g).to(cuda_device)
    f = lambda a, b, c: (_SmallAttention.apply(a, b, c, None, seed, 32 ** -0.5, 0.9) * w).sum()          # noqa: E731
    y = f(q, k, v)
    y.backward()
    assert float(f(q, k, v)) == float(y)                       # same seed -> same mask -> same value
    no_drop = _SmallAttention.apply(q, k, v, None, None, 32 ** -0.5, 1.0)
    dropped = _SmallAttention.apply(q, k, v, None, seed, 32 ** -0.5, 0.9)
    assert not torch.allclose(no_drop, dropped)
    # E[dropout(p)] = p: the mean over many elements is close
    assert abs(float((dropped - no_drop).mean())) < 0.02
    for t in (q, k, v):                                        # central differences of the masked function, fp32: loose bar
        for idx in ((3, 0, 1, 7), (40, 0, 0, 31)):
            eps = 1e-2
            tp, tm = t.detach().clone(), t.detach().clone()
            tp[idx] += eps
            tm[idx] -= eps
            args_p = [tp if x is t else x.detach() for x in (q, k, v)]
            args_m = [tm if x is t else x.detach() for x in (q, k, v)]
            num = (float(f(*args_p)) - float(f(*args_m))) / (2 * eps)
            assert abs(num - float(t.grad[idx])) < 2e-2 * max(1.0, abs(num)), (idx, num, float(t.grad[idx]))


def test_key_padding_of_the_wrong_shape_or_device_is_rejected(op, cuda_device):
    """A [L, B] (transposed) or flattened mask has the right element count but the wrong layout, and a host mask cannot
    be read by the kernel: errors in both directions, not a silently wrong pattern."""
    from trackformer_b200.small_attention import _SmallAttention
    g = torch.Generator().manual_seed(9)
    L, B, H = 40, 2, 2
    q, k, v = (torch.randn(L, B, H, 32, generator=g).to(cuda_device) for _ in range(3))
    pad = torch.zeros(B, L, dtype=torch.bool, device=cuda_device)
    pad[1, 30:] = True
    out, lse = op.small_attention_forward(q, k, v, pad, None, 32 ** -0.5, 1.0)
    op.small_attention_backward(q, k, v, pad, None, out, lse, out, 32 ** -0.5, 1.0)
    for bad in (pad.t().contiguous(), pad.flatten(), pad.cpu()):
        with pytest.raises(RuntimeError, match="key_pad"):
            _SmallAttention.apply(q, k, v, bad, None, 32 ** -0.5, 1.0)
        with pytest.raises(RuntimeError, match="key_pad"):
            op.small_attention_backward(q, k, v, bad, None, out, lse, out, 32 ** -0.5, 1.0)


def test_module_replacement_equals_stock_multihead_attention(cuda_device):
    """mha_forward(module, ...) against module(...) itself (eval mode: no dropout), outputs and parameter gradients."""
    from trackformer_b200 import small_attention
    torch.manual_seed(0)
    mha = torch.nn.MultiheadAttention(256, 8, dropout=0.1).to(cuda_device).eval()
    L, B = 300, 2
    x = torch.randn(L, B, 256, device=cuda_device, requires_grad=True)
    val = torch.randn(L, B, 256, device=cuda_device, requires_grad=True)
    pad = torch.zeros(B, L, dtype=torch.bool, device=cuda_device)
    pad[1, 250:] = True
    assert small_attention.supported(mha, x)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        gout = torch.randn(L, B, 256, device=cuda_device)
        ours = small_attention.mha_forward(mha, x, val, pad)
        ours.backward(gout)
        got = [p.grad.clone() for p in mha.parameters()] + [x.grad.clone(), val.grad.clone()]
        for p in list(mha.parameters()) + [x, val]:
            p.grad = None
        ref = mha(x, x, val, key_padding_mask=pad, need_weights=False)[0]
        ref.backward(gout)
        want = [p.grad for p in mha.parameters()] + [x.grad, val.grad]
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    torch.testing.assert_close(ours, ref, rtol=1e-4, atol=1e-5)
    for a, r in zip(got, want):
        torch.testing.assert_close(a, r, rtol=1e-3, atol=1e-4 * float(r.abs().max()))
