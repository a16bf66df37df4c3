"""The vanilla transformer's multi-head attention on the dense-attention kernels (csrc/dense_attn.cu) against an fp64
restatement of softmax(q k^T / sqrt(32) + key_pad) v: the forward and all three gradients at the encoder (1050 and 4200
tokens, DC5) and decoder cross-attention shapes, awkward sizes on both axes, strided views of a packed projection,
fully masked rows, the dropout path, bitwise reproducibility, and the nn.MultiheadAttention replacement against the
stock module with identical parameters."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SCALE = 32 ** -0.5


@pytest.fixture(scope="module")
def op(cuda_device):
    from trackformer_b200 import ext
    yield ext.load()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()          # the 4200-token fp64 references hold several GB


def _ref(q, k, v, key_pad):
    # q [Lq, B, H, 32], k / v [Lk, B, H, 32] -> [Lq, B, H, 32], in the dtype of the inputs
    qq, kk, vv = (t.permute(1, 2, 0, 3) for t in (q, k, v))
    s = qq @ kk.transpose(-1, -2) * SCALE
    if key_pad is not None:
        s = s.masked_fill(key_pad[:, None, None, :], float("-inf"))
    return (torch.softmax(s, -1) @ vv).permute(2, 0, 1, 3)


def _packed_views(Lq, Lk, B, H, g, device):
    """q from one packed [Lq, B, H*32] projection, k and v strided views of one packed [Lk, B, 2*H*32] projection
    (the layout of the in-projection outputs the module consumes in place)."""
    e = H * 32
    pq = torch.randn(Lq, B, e, generator=g).to(device)
    pkv = torch.randn(Lk, B, 2 * e, generator=g).to(device)
    q = pq.unflatten(-1, (H, 32))
    k, v = pkv[..., :e].unflatten(-1, (H, 32)), pkv[..., e:].unflatten(-1, (H, 32))
    return [t.detach().requires_grad_(True) for t in (q, k, v)]


def _image_padding(B, hw, valid, device):
    """[B, h*w] key padding of a batch of images padded on the right and bottom (scattered in flattened order)."""
    h, w = hw
    pad = torch.ones(B, h, w, dtype=torch.bool, device=device)
    for i, (vh, vw) in enumerate(valid):
        pad[i, :vh, :vw] = False
    return pad.flatten(1)


def _check(q, k, v, key_pad, g, rtol=1e-4, atol=1e-5, gatol=2e-5):
    from trackformer_b200.dense_attention import _DenseAttention
    out = _DenseAttention.apply(q, k, v, key_pad, None, SCALE, 1.0)
    gout = torch.randn(out.shape, generator=g).to(out.device)
    out.backward(gout)
    qr, kr, vr = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = _ref(qr, kr, vr, key_pad)
    ref.backward(gout.double())
    torch.testing.assert_close(out.double(), ref, rtol=rtol, atol=atol)
    for name, a, r in (("dq", q, qr), ("dk", k, kr), ("dv", v, vr)):
        torch.testing.assert_close(a.grad.double(), r.grad, rtol=rtol, atol=gatol, msg=lambda m: f"{name}: {m}")


@pytest.mark.parametrize("hw,valid", [((25, 42), [(25, 42), (19, 33)]), ((50, 84), [(44, 84), (50, 61)])],
                         ids=["1050", "4200"])
def test_encoder_self_attention_matches_fp64(op, cuda_device, hw, valid):
    g = torch.Generator().manual_seed(hw[0])
    L = hw[0] * hw[1]
    packed = torch.randn(L, 2, 3 * 256, generator=g).to(cuda_device)
    q, k, v = (packed[..., i * 256:(i + 1) * 256].unflatten(-1, (8, 32)).detach().requires_grad_(True) for i in range(3))
    _check(q, k, v, _image_padding(2, hw, valid, cuda_device), g)


@pytest.mark.parametrize("Lq", [100, 137, 300])
def test_decoder_cross_attention_matches_fp64(op, cuda_device, Lq):
    g = torch.Generator().manual_seed(Lq)
    q, k, v = _packed_views(Lq, 1050, 2, 8, g, cuda_device)
    _check(q, k, v, _image_padding(2, (25, 42), [(25, 42), (21, 30)], cuda_device), g)


@pytest.mark.parametrize("Lq", [1, 33, 65, 129])
@pytest.mark.parametrize("Lk", [1, 33, 65, 129])
def test_awkward_sizes_match_fp64(op, cuda_device, Lq, Lk):
    g = torch.Generator().manual_seed(1000 * Lq + Lk)
    q, k, v = _packed_views(Lq, Lk, 3, 2, g, cuda_device)
    key_pad = None
    if Lk > 1:
        key_pad = torch.rand(3, Lk, generator=g).to(cuda_device) < 0.3
        key_pad[:, 0] = False                          # every row keeps a key: the fp64 softmax is defined
    _check(q, k, v, key_pad, g)


def test_fully_masked_rows_give_zero_output_and_gradients(op, cuda_device):
    from trackformer_b200.dense_attention import _DenseAttention
    g = torch.Generator().manual_seed(3)
    q, k, v = _packed_views(70, 130, 2, 2, g, cuda_device)
    key_pad = torch.zeros(2, 130, dtype=torch.bool, device=cuda_device)
    key_pad[1] = True
    key_pad[0, 5:77] = True
    out = _DenseAttention.apply(q, k, v, key_pad, None, SCALE, 1.0)
    out.backward(torch.randn(out.shape, generator=g).to(cuda_device))
    assert torch.isfinite(out).all()
    assert (out[:, 1] == 0).all() and (q.grad[:, 1] == 0).all() and (k.grad[:, 1] == 0).all() and (v.grad[:, 1] == 0).all()
    assert (k.grad[5:77, 0] == 0).all() and (v.grad[5:77, 0] == 0).all()
    qr, kr, vr = (t.detach()[:, :1].double() for t in (q, k, v))
    torch.testing.assert_close(out[:, :1].double(), _ref(qr, kr, vr, key_pad[:1]), rtol=1e-4, atol=1e-5)


def test_dropout_is_deterministic_and_differentiated_consistently(op, cuda_device):
    from trackformer_b200.dense_attention import _DenseAttention
    g = torch.Generator().manual_seed(5)
    Lq, Lk, B, H = 40, 150, 1, 2
    q = torch.randn(Lq, B, H, 32, generator=g).to(cuda_device).requires_grad_(True)
    k, v = (torch.randn(Lk, B, H, 32, generator=g).to(cuda_device).requires_grad_(True) for _ in range(2))
    seed = torch.tensor([1234567], dtype=torch.int64, device=cuda_device)
    w = torch.randn(Lq, B, H, 32, generator=g).to(cuda_device)
    f = lambda a, b, c: (_DenseAttention.apply(a, b, c, None, seed, SCALE, 0.9) * w).sum()          # noqa: E731
    y = f(q, k, v)
    y.backward()
    assert float(f(q, k, v)) == float(y)                       # same seed -> same mask -> same value
    for t in (q, k, v):                                        # central differences of the masked function, fp32
        for idx in ((3, 0, 1, 7), (37, 0, 0, 31)):
            eps = 1e-2
            tp, tm = t.detach().clone(), t.detach().clone()
            tp[idx] += eps
            tm[idx] -= eps
            args_p = [tp if x is t else x.detach() for x in (q, k, v)]
            args_m = [tm if x is t else x.detach() for x in (q, k, v)]
            num = (float(f(*args_p)) - float(f(*args_m))) / (2 * eps)
            assert abs(num - float(t.grad[idx])) < 2e-2 * max(1.0, abs(num)), (idx, num, float(t.grad[idx]))


def test_dropout_mask_statistics(op, cuda_device):
    """E[dropout(P) V] = P V: over many elements the mean difference vanishes; and the kept share of the attention
    weights is keep_prob (read off with V = one-hot columns, so that out = dropout(P) restricted to 32 keys)."""
    from trackformer_b200.dense_attention import _DenseAttention
    g = torch.Generator().manual_seed(6)
    Lq, Lk, B, H = 500, 32, 2, 8
    q = torch.randn(Lq, B, H, 32, generator=g).to(cuda_device)
    k = torch.randn(Lk, B, H, 32, generator=g).to(cuda_device)
    v = torch.eye(32, device=cuda_device)[:, None, None, :].expand(Lk, B, H, 32).contiguous()
    seed = torch.tensor([42], dtype=torch.int64, device=cuda_device)
    no_drop = _DenseAttention.apply(q, k, v, None, None, SCALE, 1.0)
    dropped = _DenseAttention.apply(q, k, v, None, seed, SCALE, 0.9)
    kept = dropped != 0
    assert abs(float(kept.double().mean()) - 0.9) < 0.01
    torch.testing.assert_close(dropped[kept], no_drop[kept] / 0.9, rtol=1e-5, atol=1e-7)
    assert abs(float((dropped - no_drop).sum(-1).mean())) < 0.01


def test_gradients_are_bitwise_reproducible(op, cuda_device):
    from trackformer_b200.dense_attention import _DenseAttention
    g = torch.Generator().manual_seed(8)
    q, k, v = _packed_views(300, 1050, 2, 8, g, cuda_device)
    key_pad = _image_padding(2, (25, 42), [(25, 42), (20, 31)], cuda_device)
    seed = torch.tensor([99], dtype=torch.int64, device=cuda_device)
    gout = torch.randn(300, 2, 8, 32, generator=g).to(cuda_device)
    runs = []
    for _ in range(2):
        for t in (q, k, v):
            t.grad = None
        _DenseAttention.apply(q, k, v, key_pad, seed, SCALE, 0.9).backward(gout)
        runs.append([t.grad.clone() for t in (q, k, v)])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def _module_case(cuda_device, Lq, Lk, cross):
    """mha_forward(module, ...) against module(...) itself (eval mode: no dropout), outputs and every gradient."""
    from trackformer_b200 import dense_attention
    torch.manual_seed(Lq + Lk)
    mha = torch.nn.MultiheadAttention(256, 8, dropout=0.1).to(cuda_device).eval()
    B = 2
    tgt = torch.randn(Lq, B, 256, device=cuda_device, requires_grad=True)
    qpos = torch.randn(Lq, B, 256, device=cuda_device)
    memory = torch.randn(Lk, B, 256, device=cuda_device, requires_grad=True)
    pos = torch.randn(Lk, B, 256, device=cuda_device)
    pad = _image_padding(B, (25, 42), [(25, 42), (18, 37)], cuda_device) if Lk == 1050 else None
    leaves = [tgt, memory]

    def run(fn):
        q = tgt + qpos
        if cross:
            return fn(q, memory + pos, memory, pad)
        x = memory + pos
        return fn(x, x, memory, pad)

    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        assert dense_attention.supported(mha, tgt)
        gout = torch.randn(Lq if cross else Lk, B, 256, device=cuda_device)
        ours = run(lambda q, k, v, m: dense_attention.mha_forward(mha, q, k, v, m))
        ours.backward(gout)
        got = [p.grad.clone() for p in mha.parameters()] + [t.grad.clone() for t in leaves if t.grad is not None]
        for p in list(mha.parameters()) + leaves:
            p.grad = None
        ref = run(lambda q, k, v, m: mha(q, k, v, key_padding_mask=m, need_weights=False)[0])
        ref.backward(gout)
        want = [p.grad for p in mha.parameters()] + [t.grad for t in leaves if t.grad is not None]
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    torch.testing.assert_close(ours, ref, rtol=1e-4, atol=1e-5)
    assert len(got) == len(want)
    for a, r in zip(got, want):
        torch.testing.assert_close(a, r, rtol=1e-3, atol=1e-4 * float(r.abs().max()))


def test_module_replacement_encoder_self_attention(op, cuda_device):
    _module_case(cuda_device, 1050, 1050, cross=False)


@pytest.mark.parametrize("Lq", [100, 137])
def test_module_replacement_decoder_cross_attention(op, cuda_device, Lq):
    _module_case(cuda_device, Lq, 1050, cross=True)


def test_key_padding_of_the_wrong_shape_is_rejected(op, cuda_device):
    """A [Lk, B] (transposed) or flattened mask has the right element count but the wrong layout: an error, not a
    silently wrong pattern."""
    from trackformer_b200.dense_attention import _DenseAttention
    g = torch.Generator().manual_seed(9)
    q, k, v = _packed_views(16, 40, 2, 2, g, cuda_device)
    pad = torch.zeros(2, 40, dtype=torch.bool, device=cuda_device)
    _DenseAttention.apply(q, k, v, pad, None, SCALE, 1.0)
    for bad in (pad.t().contiguous(), pad.flatten()):
        with pytest.raises(RuntimeError, match="key_pad"):
            _DenseAttention.apply(q, k, v, bad, None, SCALE, 1.0)
