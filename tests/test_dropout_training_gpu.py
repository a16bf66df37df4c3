"""Training mode with dropout 0.1 (cfgs/train.yaml) pinned to fp64 restatements that replay the kernels' own masks.

Every fused dropout site draws one int64 seed from trackformer_b200/seeds.py and keeps element idx iff a hash of
(seed, idx) falls below keep * 2^32; tests/dropout_hash.py restates that hash on the host.  So the masks of a training
pass can be rebuilt bit for bit and training mode compared as tightly as eval mode:

* kernel level -- the kept sets of relu_dropout, the seeded residual + LayerNorm and both attention kernels equal the
  restatement bitwise (tails on every axis), and the forward and every gradient equal fp64 with the restated mask at
  the production shapes;
* layer level -- the deformable and vanilla encoder / decoder layers (post- and pre-norm) in train mode against fp64
  restatements of the reference's own forward (models/deformable_transformer.py:282-293, 358-380;
  models/transformer.py:188-215, 251-295), consuming the recorded seeds in the reference's site order and the masks of
  the stock nn.Dropout sites captured by forward hooks; then the whole vanilla Transformer;
* seeds and CUDA graphs -- one seed per fused site per pass, all distinct and drawn from the pool; a graphed TrainStep
  equals the eager one under the same (deterministic, captured) seeds, and draws fresh masks on every replay.
"""
import copy
import math

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import dropout_hash as dh

pytestmark = pytest.mark.gpu

SCALE = 32 ** -0.5
P_DROP = 0.1
KEEP = 1.0 - P_DROP
SEEDS = [0x2F3A5B7C9D1E0F21, 12345, (1 << 32) + 1]


@pytest.fixture(scope="module", autouse=True)
def _free_cache_at_teardown():
    yield
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()      # the 4200-token and C2 fp64 references hold several GB


@pytest.fixture(scope="module")
def op(cuda_device):
    from trackformer_b200 import ext
    return ext.load()


@pytest.fixture()
def strict_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _seed_tensor(seed, device):
    return torch.tensor([seed], dtype=torch.int64, device=device)


def _close(name, got, want, rtol, rel_atol):
    scale = float(want.abs().max()) or 1.0
    torch.testing.assert_close(got.double(), want, rtol=rtol, atol=rel_atol * scale, msg=lambda m: f"{name}: {m}")


def _image_padding(B, hw, valid, device):
    """[B, h*w] key padding of a batch of images padded on the right and bottom."""
    h, w = hw
    pad = torch.ones(B, h, w, dtype=torch.bool, device=device)
    for i, (vh, vw) in enumerate(valid):
        pad[i, :vh, :vw] = False
    return pad.flatten(1)


# ------------------------------------------------------------------------------------------------------------------
# 3a. kernel level: the kept sets equal the restatement bit for bit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(22223, 1024), (3 * 132 * 16 * 256 * 4 + 148,), (4100,)],
                         ids=["c2_ffn", "grid_stride_tail", "one_partial_cta"])
def test_relu_dropout_mask_is_the_restated_hash(op, cuda_device, shape):
    g = torch.Generator().manual_seed(len(shape))
    a = (torch.randn(shape, generator=g).abs() + 1e-3).to(cuda_device)     # all positive: h != 0 <=> kept
    for seed in SEEDS:
        h = op.relu_dropout_forward(a, _seed_tensor(seed, cuda_device), KEEP, True)
        want = dh.relu_dropout_mask(seed, shape, KEEP, cuda_device)
        got = h != 0
        assert torch.equal(got, want), f"seed {seed:#x}: {int((got != want).sum())} elements disagree"
    # negative inputs are never resurrected, whatever the mask
    h = op.relu_dropout_forward(-a, _seed_tensor(SEEDS[0], cuda_device), KEEP, True)
    assert not bool(h.any())


@pytest.mark.parametrize("rows,C,p", [(22223, 256, 0.1), (4097, 288, 0.3), (33, 128, 0.5)])
def test_seeded_layernorm_mask_is_the_restated_hash(op, cuda_device, rows, C, p):
    g = torch.Generator().manual_seed(rows + C)
    x = torch.zeros(rows, C, device=cuda_device)                             # s = x + dropout(branch) = dropout(branch)
    br = torch.randn(rows, C, generator=g)
    br[br == 0] = 1.0
    br = br.to(cuda_device)
    gamma, beta = torch.ones(C, device=cuda_device), torch.zeros(C, device=cuda_device)
    for seed in SEEDS:
        s = op.add_dropout_layernorm_seeded_forward(x, br, _seed_tensor(seed, cuda_device), gamma, beta, 1.0 - p, 1e-5)[1]
        want = dh.layernorm_mask(seed, rows, C, 1.0 - p, cuda_device)
        got = s != 0
        assert torch.equal(got, want), f"seed {seed:#x}: {int((got != want).sum())} elements disagree"


def _read_attention_keep(fwd, q, k, key_pad, seed, keep):
    """Kept set [B, H, Lq, Lk] of a kernel's attention dropout, read off with one-hot V blocks: with V = e_j on key
    k0 + j, output channel j is dropout(P)[q, k0 + j] / rowsum(P), > 0 iff that weight was kept."""
    Lk, B, H, _ = k.shape
    Lq = q.shape[0]
    kept = torch.zeros(B, H, Lq, Lk, dtype=torch.bool, device=q.device)
    eye = torch.eye(32, device=q.device)
    for k0 in range(0, Lk, 32):
        n = min(32, Lk - k0)
        v = torch.zeros(Lk, B, H, 32, device=q.device)
        v[k0:k0 + n] = eye[:n, None, None, :]
        out = fwd(q, k, v, key_pad, _seed_tensor(seed, q.device), SCALE, keep)[0]
        kept[..., k0:k0 + n] = (out[..., :n] > 0).permute(1, 2, 0, 3)
    return kept


def _expected_attention_keep(seed, B, H, Lq, Lk, keep, key_pad, device):
    want = dh.attention_mask(seed, B, H, Lq, Lk, keep, device)
    if key_pad is not None:
        want &= ~key_pad[:, None, None, :]
    return want


@pytest.mark.parametrize("L", [33, 77, 300])
def test_small_attention_mask_is_the_restated_hash(op, cuda_device, L):
    g = torch.Generator().manual_seed(L)
    B, H = 2, 8
    q, k = (0.3 * torch.randn(L, B, H, 32, generator=g)).to(cuda_device), torch.randn(L, B, H, 32, generator=g).to(cuda_device)
    key_pad = torch.zeros(B, L, dtype=torch.bool, device=cuda_device)
    key_pad[1, L - L // 4:] = True
    key_pad[0, 5] = True
    for seed in SEEDS[:2]:
        got = _read_attention_keep(op.small_attention_forward, q, k, key_pad, seed, KEEP)
        want = _expected_attention_keep(seed, B, H, L, L, KEEP, key_pad, cuda_device)
        assert torch.equal(got, want), f"seed {seed:#x}: {int((got != want).sum())} weights disagree"


@pytest.mark.parametrize("Lq", [1, 65, 100])
@pytest.mark.parametrize("Lk", [33, 129, 1050])
def test_dense_attention_mask_is_the_restated_hash(op, cuda_device, Lq, Lk):
    g = torch.Generator().manual_seed(1000 * Lq + Lk)
    B, H = 2, 8
    q = (0.3 * torch.randn(Lq, B, H, 32, generator=g)).to(cuda_device)
    k = torch.randn(Lk, B, H, 32, generator=g).to(cuda_device)
    if Lk == 1050:
        key_pad = _image_padding(B, (25, 42), [(25, 42), (19, 33)], cuda_device)
    else:
        hw = (3, Lk // 3)
        key_pad = _image_padding(B, hw, [hw, (2, hw[1] - 4)], cuda_device)
    seed = SEEDS[0]
    got = _read_attention_keep(op.dense_attention_forward, q, k, key_pad, seed, KEEP)
    want = _expected_attention_keep(seed, B, H, Lq, Lk, KEEP, key_pad, cuda_device)
    assert torch.equal(got, want), f"{int((got != want).sum())} weights disagree"


# ------------------------------------------------------------------------------------------------------------------
# 3b. kernel level: forward and every gradient against fp64 with the restated mask
# ------------------------------------------------------------------------------------------------------------------
def _attention_fp64(q, k, v, key_pad, keep_mask, keep):
    qq, kk, vv = (t.permute(1, 2, 0, 3) for t in (q, k, v))
    s = qq @ kk.transpose(-1, -2) * SCALE
    if key_pad is not None:
        s = s.masked_fill(key_pad[:, None, None, :], float("-inf"))
    a = torch.softmax(s, -1) * keep_mask / keep
    return (a @ vv).permute(2, 0, 1, 3)


def _check_attention_with_dropout(fn, q, k, v, key_pad, seed, g):
    Lq, B, H, _ = q.shape
    Lk = k.shape[0]
    out = fn(q, k, v, key_pad, _seed_tensor(seed, q.device), SCALE, KEEP)
    gout = torch.randn(out.shape, generator=g).to(out.device)
    out.backward(gout)
    mask = dh.attention_mask(seed, B, H, Lq, Lk, KEEP, q.device)
    qr, kr, vr = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = _attention_fp64(qr, kr, vr, key_pad, mask, KEEP)
    del mask
    ref.backward(gout.double())
    _close("out", out.detach(), ref.detach(), 1e-4, 1e-5)
    for name, a, r in (("dq", q, qr), ("dk", k, kr), ("dv", v, vr)):
        _close(name, a.grad, r.grad, 1e-4, 2e-5)


@pytest.mark.parametrize("hw,valid", [((25, 42), [(25, 42), (19, 33)]), ((50, 84), [(44, 84), (50, 61)])],
                         ids=["1050", "4200"])
def test_dense_encoder_attention_with_dropout_matches_fp64(op, cuda_device, hw, valid):
    from trackformer_b200.dense_attention import _DenseAttention
    g = torch.Generator().manual_seed(hw[0] + 1)
    L = hw[0] * hw[1]
    packed = torch.randn(L, 2, 3 * 256, generator=g).to(cuda_device)
    q, k, v = (packed[..., i * 256:(i + 1) * 256].unflatten(-1, (8, 32)).detach().requires_grad_(True) for i in range(3))
    _check_attention_with_dropout(_DenseAttention.apply, q, k, v, _image_padding(2, hw, valid, cuda_device), SEEDS[0], g)


@pytest.mark.parametrize("Lq", [100, 137])
def test_dense_cross_attention_with_dropout_matches_fp64(op, cuda_device, Lq):
    from trackformer_b200.dense_attention import _DenseAttention
    g = torch.Generator().manual_seed(Lq + 7)
    q = torch.randn(Lq, 2, 8, 32, generator=g).to(cuda_device).requires_grad_(True)
    pkv = torch.randn(1050, 2, 512, generator=g).to(cuda_device)
    k, v = (pkv[..., i * 256:(i + 1) * 256].unflatten(-1, (8, 32)).detach().requires_grad_(True) for i in range(2))
    key_pad = _image_padding(2, (25, 42), [(25, 42), (21, 30)], cuda_device)
    _check_attention_with_dropout(_DenseAttention.apply, q, k, v, key_pad, SEEDS[1], g)


@pytest.mark.parametrize("L,filler", [(300, 0), (400, 60)], ids=["300_queries", "400_rows_60_filler"])
def test_small_attention_with_dropout_matches_fp64(op, cuda_device, L, filler):
    """Filler rows (the fixed-shape track-query padding of GraphedDetector) are hidden as keys; every row, filler rows
    included, must still equal the fp64 restatement."""
    from trackformer_b200.small_attention import _SmallAttention
    g = torch.Generator().manual_seed(L + filler)
    packed = torch.randn(L, 2, 3 * 256, generator=g).to(cuda_device)
    q, k, v = (packed[..., i * 256:(i + 1) * 256].unflatten(-1, (8, 32)).detach().requires_grad_(True) for i in range(3))
    key_pad = None
    if filler:
        key_pad = torch.zeros(2, L, dtype=torch.bool, device=cuda_device)
        key_pad[:, L - filler:] = True
    _check_attention_with_dropout(_SmallAttention.apply, q, k, v, key_pad, SEEDS[2], g)


def test_relu_dropout_forward_backward_match_fp64(op, cuda_device):
    g = torch.Generator().manual_seed(1)
    a = torch.randn(22223, 1024, generator=g).to(cuda_device)
    gh = torch.randn(22223, 1024, generator=g).to(cuda_device)
    seed = SEEDS[0]
    h = op.relu_dropout_forward(a, _seed_tensor(seed, cuda_device), KEEP, True)
    ga = op.relu_dropout_backward(gh, h, KEEP, True)
    mask = dh.relu_dropout_mask(seed, a.shape, KEEP, cuda_device)
    ad = a.double()
    live = (ad > 0) & mask
    torch.testing.assert_close(h.double(), torch.where(live, ad / KEEP, 0.0), rtol=1e-6, atol=0)
    torch.testing.assert_close(ga.double(), torch.where(live, gh.double() / KEEP, 0.0), rtol=1e-6, atol=0)


@pytest.mark.parametrize("rows,C,p", [(22223, 256, 0.1), (4097, 288, 0.3)])
def test_seeded_layernorm_forward_backward_match_fp64(op, cuda_device, rows, C, p):
    """All four gradients of norm(x + dropout(branch)) against fp64 with the restated mask: the backward recomputes the
    mask from the seed, so an index slip there shows up in dbranch even when the forward is right."""
    g = torch.Generator().manual_seed(rows * 3 + C)
    x, br, dy = (torch.randn(rows, C, generator=g).to(cuda_device) for _ in range(3))
    gamma = (torch.rand(C, generator=g) + 0.5).to(cuda_device)
    beta = torch.randn(C, generator=g).to(cuda_device)
    keep, seed = 1.0 - p, SEEDS[0]
    st = _seed_tensor(seed, cuda_device)
    y, s, mean, rstd = op.add_dropout_layernorm_seeded_forward(x, br, st, gamma, beta, keep, 1e-5)
    dx, dbr, dgamma, dbeta = op.add_dropout_layernorm_seeded_backward(dy, s, st, gamma, mean, rstd, keep)
    mask = dh.layernorm_mask(seed, rows, C, keep, cuda_device)
    xr, brr, gr, btr = (t.double().requires_grad_(True) for t in (x, br, gamma, beta))
    y_ref = F.layer_norm(xr + brr * mask / keep, (C,), gr, btr, 1e-5)
    y_ref.backward(dy.double())
    _close("y", y, y_ref.detach(), 1e-4, 1e-5)
    _close("dx", dx, xr.grad, 1e-4, 1e-5)
    _close("dbranch", dbr, brr.grad, 1e-4, 1e-5)
    _close("dgamma", dgamma, gr.grad, 1e-4, 1e-5)
    _close("dbeta", dbeta, btr.grad, 1e-4, 1e-5)


# ------------------------------------------------------------------------------------------------------------------
# 4. layer level: train mode against fp64 restatements of the reference's layers
# ------------------------------------------------------------------------------------------------------------------
class _Recorder:
    """Seeds handed out by ``seeds.next_seed`` (call order) and the masks of the stock nn.Dropout modules that ran."""

    def __init__(self, monkeypatch, model):
        from trackformer_b200 import deformable_transformer, fused_linear, seeds, transformer
        self.drawn, self.stock, self.relu_signs = [], {}, []
        orig = seeds.next_seed

        def next_seed(device):
            s = orig(device)
            self.drawn.append(s)
            return s
        monkeypatch.setattr(seeds, "next_seed", next_seed)

        def relu_dropout(a, dropout):
            # the side of the ReLU kink the fp32 pass took: where |a| is at rounding level fp64 may take the other
            # one, and the gradient of that whole row would differ for a reason that has nothing to do with dropout
            self.relu_signs.append(a.detach() > 0)
            return fused_linear.relu_dropout(a, dropout)
        for mod in (transformer, deformable_transformer):
            monkeypatch.setattr(mod, "relu_dropout", relu_dropout)
        self.handles = []
        for name, m in model.named_modules():
            if isinstance(m, nn.Dropout):
                self.handles.append(m.register_forward_hook(
                    lambda mod, inp, out, name=name: self.stock.__setitem__(name, out.detach() != 0)))

    def replay(self):
        for h in self.handles:
            h.remove()
        return _Replay([int(s.item()) for s in self.drawn], self.stock, self.relu_signs)


class _Replay:
    """Hands the recorded seeds and stock masks to the fp64 restatement in the reference's site order."""

    def __init__(self, seed_values, stock, relu_signs=None):
        self.seeds, self.stock = list(seed_values), dict(stock)
        self.relu_signs = list(relu_signs) if relu_signs is not None else None
        self.n_seeds = len(self.seeds)
        self.used_seeds, self.used_stock = 0, set()

    def seed(self):
        assert self.used_seeds < self.n_seeds, "the reference has more fused dropout sites than seeds were drawn"
        self.used_seeds += 1
        return self.seeds[self.used_seeds - 1]

    def fused(self, x, branch, p):
        """dropout(branch) at a fused residual site (mask over x's logical layout)."""
        return branch * dh.keep_mask(self.seed(), x.shape, 1.0 - p, x.device) / (1.0 - p)

    def relu(self, a, p):
        if self.relu_signs is None:
            act = F.relu(a)
        else:
            assert self.relu_signs, "the reference has more FFN activations than relu_dropout ran"
            act = torch.where(self.relu_signs.pop(0), a, 0.0)
        return act * dh.keep_mask(self.seed(), a.shape, 1.0 - p, a.device) / (1.0 - p)

    def attention(self, B, H, Lq, Lk, p, device):
        return dh.attention_mask(self.seed(), B, H, Lq, Lk, 1.0 - p, device)

    def stock_dropout(self, name, x, p):
        assert name in self.stock, f"{name}: the reference applies dropout here, the module under test did not"
        self.used_stock.add(name)
        return x * self.stock[name] / (1.0 - p)

    def done(self):
        assert self.used_seeds == self.n_seeds, f"{self.n_seeds} seeds drawn, the reference consumed {self.used_seeds}"
        extra = set(self.stock) - self.used_stock
        assert not extra, f"stock dropout ran where the reference has none: {sorted(extra)}"
        assert not self.relu_signs, "relu_dropout ran where the reference has no FFN activation"


def _params64(module):
    return {k: v.detach().double().requires_grad_(True) for k, v in module.named_parameters()}


def _perturb_(module, seed):
    """Move every parameter off its init (zero offset / logit weights, unit norms) so that each one is exercised."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            p.add_(torch.randn(p.shape, generator=g).to(p.device) * (0.1 if "norm" in name else 0.02))


def _lin(P, pre, x):
    return x @ P[pre + "weight"].t() + P[pre + "bias"]


def _ln(P, pre, x):
    return F.layer_norm(x, (x.shape[-1],), P[pre + "weight"], P[pre + "bias"], 1e-5)


def _mha(P, pre, query, key, value, key_pad, rp, p):
    """nn.MultiheadAttention (sequence first, 32 channels per head) spelled out: in-projection split, q scaling, softmax,
    dropout on the weights, @ v, out-projection."""
    E = query.shape[-1]
    H = E // 32
    W, b = P[pre + "in_proj_weight"], P[pre + "in_proj_bias"]
    q = (query @ W[:E].t() + b[:E]) * (E // H) ** -0.5
    k = key @ W[E:2 * E].t() + b[E:2 * E]
    v = value @ W[2 * E:].t() + b[2 * E:]
    Lq, B, _ = q.shape
    Lk = k.shape[0]
    q, k, v = (t.reshape(t.shape[0], B, H, 32).permute(1, 2, 0, 3) for t in (q, k, v))
    s = q @ k.transpose(-1, -2)
    if key_pad is not None:
        s = s.masked_fill(key_pad[:, None, None, :], float("-inf"))
    a = torch.softmax(s, -1)
    a = a * rp.attention(B, H, Lq, Lk, p, query.device) / (1.0 - p)
    o = (a @ v).permute(2, 0, 1, 3).reshape(Lq, B, E)
    return o @ P[pre + "out_proj.weight"].t() + P[pre + "out_proj.bias"]


def _msda(P, pre, query, ref, value_in, hw, pad, heads=8, levels=4, points=4):
    """MSDeformAttn.forward of the reference (ops/modules/ms_deform_attn.py:60-89) in fp64, core by msda_core_torch."""
    from oracle.torch_ref import msda_core_torch
    N, Lq, C = query.shape
    S = value_in.shape[1]
    value = _lin(P, pre + "value_proj.", value_in)
    if pad is not None:
        value = value.masked_fill(pad[..., None], 0.0)
    value = value.view(N, S, heads, C // heads)
    off = _lin(P, pre + "sampling_offsets.", query).view(N, Lq, heads, levels, points, 2)
    aw = F.softmax(_lin(P, pre + "attention_weights.", query).view(N, Lq, heads, levels * points), -1)
    aw = aw.view(N, Lq, heads, levels, points)
    if ref.shape[-1] == 2:
        shapes = torch.tensor(hw, dtype=torch.float64, device=query.device)        # (H, W) as stored, like the reference
        loc = ref[:, :, None, :, None, :] + off / shapes[None, None, None, :, None, :]
    else:
        loc = ref[:, :, None, :, None, :2] + off / points * ref[:, :, None, :, None, 2:] * 0.5
    return _lin(P, pre + "output_proj.", msda_core_torch(value, hw, loc, aw))


def _deformable_encoder_layer_ref(P, pre, src, pos, ref, hw, pad, rp, p):
    """models/deformable_transformer.py:282-297."""
    src2 = _msda(P, pre + "self_attn.", src + pos, ref, src, hw, pad)
    src = _ln(P, pre + "norm1.", src + rp.fused(src, src2, p))                                     # dropout1
    src2 = _lin(P, pre + "linear2.", rp.relu(_lin(P, pre + "linear1.", src), p))                   # dropout2
    return _ln(P, pre + "norm2.", src + rp.fused(src, src2, p))                                    # dropout3


def _deformable_decoder_layer_ref(P, pre, tgt, qpos, ref, src, hw, src_pad, key_pad, rp, p):
    """models/deformable_transformer.py:358-383, the query padding applied as the self-attention key padding."""
    q = (tgt + qpos).transpose(0, 1)
    tgt2 = _mha(P, pre + "self_attn.", q, q, tgt.transpose(0, 1), key_pad, rp, p).transpose(0, 1)
    tgt = _ln(P, pre + "norm2.", tgt + rp.fused(tgt, tgt2, p))                                     # dropout2
    tgt2 = _msda(P, pre + "cross_attn.", tgt + qpos, ref, src, hw, src_pad)
    tgt = _ln(P, pre + "norm1.", tgt + rp.fused(tgt, tgt2, p))                                     # dropout1
    h = rp.stock_dropout(pre + "dropout3", F.relu(_lin(P, pre + "linear1.", tgt)), p)
    return _ln(P, pre + "norm3.", tgt + rp.fused(tgt, _lin(P, pre + "linear2.", h), p))           # dropout4


def _encoder_layer_ref(P, pre, src, pad, pos, pre_norm, rp, p):
    """models/transformer.py:188-215."""
    if not pre_norm:
        qk = src + pos
        src = _ln(P, pre + "norm1.", src + rp.fused(src, _mha(P, pre + "self_attn.", qk, qk, src, pad, rp, p), p))
        src2 = _lin(P, pre + "linear2.", rp.relu(_lin(P, pre + "linear1.", src), p))
        return _ln(P, pre + "norm2.", src + rp.fused(src, src2, p))
    src2 = _ln(P, pre + "norm1.", src)
    qk = src2 + pos
    src = src + rp.stock_dropout(pre + "dropout1", _mha(P, pre + "self_attn.", qk, qk, src2, pad, rp, p), p)
    src2 = _lin(P, pre + "linear2.", rp.relu(_lin(P, pre + "linear1.", _ln(P, pre + "norm2.", src)), p))
    return src + rp.stock_dropout(pre + "dropout2", src2, p)


def _decoder_layer_ref(P, pre, tgt, memory, tgt_pad, mem_pad, pos, qpos, pre_norm, rp, p):
    """models/transformer.py:251-295."""
    if not pre_norm:
        q = tgt + qpos
        tgt = _ln(P, pre + "norm1.", tgt + rp.fused(tgt, _mha(P, pre + "self_attn.", q, q, tgt, tgt_pad, rp, p), p))
        tgt2 = _mha(P, pre + "multihead_attn.", tgt + qpos, memory + pos, memory, mem_pad, rp, p)
        tgt = _ln(P, pre + "norm2.", tgt + rp.fused(tgt, tgt2, p))
        tgt2 = _lin(P, pre + "linear2.", rp.relu(_lin(P, pre + "linear1.", tgt), p))
        return _ln(P, pre + "norm3.", tgt + rp.fused(tgt, tgt2, p))
    tgt2 = _ln(P, pre + "norm1.", tgt)
    q = tgt2 + qpos
    tgt = tgt + rp.stock_dropout(pre + "dropout1", _mha(P, pre + "self_attn.", q, q, tgt2, tgt_pad, rp, p), p)
    tgt2 = _ln(P, pre + "norm2.", tgt)
    tgt2 = _mha(P, pre + "multihead_attn.", tgt2 + qpos, memory + pos, memory, mem_pad, rp, p)
    tgt = tgt + rp.stock_dropout(pre + "dropout2", tgt2, p)
    tgt2 = _lin(P, pre + "linear2.", rp.relu(_lin(P, pre + "linear1.", _ln(P, pre + "norm3.", tgt)), p))
    return tgt + rp.stock_dropout(pre + "dropout3", tgt2, p)


def _close_but_for_kinks(name, got, want, rtol, rel_atol, max_frac):
    """Elementwise closeness on all but a ``max_frac`` share of the elements, and 1e-2 relative L2 error overall.  For
    the query-side input gradient of MSDeformAttn: a sample whose fp32 location lies within rounding of a pixel
    boundary takes the bilinear location gradient of the neighbouring cell, which moves that query's whole row.  A
    dropout mask error moves ~10 % of the elements."""
    got = got.double()
    err = (got - want).abs()
    bad = err > rel_atol * float(want.abs().max()) + rtol * want.abs()
    frac = float(bad.double().mean())
    assert frac <= max_frac, f"{name}: {int(bad.sum())} elements ({frac:.2e}) out of tolerance, max error {float(err.max())}"
    rel_l2 = float(torch.linalg.vector_norm(got - want) / torch.linalg.vector_norm(want))
    assert rel_l2 < 1e-2, f"{name}: relative L2 error {rel_l2}"


def _compare_layer(module, P, inputs, refs, out, ref_out, rtol, rel_atol, param_rel_atol, loose=(), kinked=()):
    _close("output", out.detach(), ref_out.detach(), rtol, rel_atol)
    for name, t in inputs.items():
        if name in kinked:
            _close_but_for_kinks(f"grad {name}", t.grad, refs[name].grad, rtol, rel_atol, 1e-3)
        else:
            _close(f"grad {name}", t.grad, refs[name].grad, rtol, rel_atol)
    for name, prm in module.named_parameters():
        tol = 10 * param_rel_atol if any(s in name for s in loose) else param_rel_atol
        _close(f"grad {name}", prm.grad, P[name].grad, 10 * rtol, tol)


C2_HW = [(100, 167), (50, 84), (25, 42), (13, 21)]          # 800 x 1333 at strides 8..64: 22223 tokens


def _level_padding(hw, B, device):
    """[B, S] padding of a batch whose second image covers ~80 % x 70 % of every level, and its valid ratios."""
    masks, ratios = [], []
    for h, w in hw:
        m = torch.zeros(B, h, w, dtype=torch.bool, device=device)
        vh, vw = math.ceil(0.8 * h), math.ceil(0.7 * w)
        m[1, vh:] = True
        m[1, :, vw:] = True
        masks.append(m.flatten(1))
        ratios.append(torch.tensor([[1.0, 1.0], [vw / w, vh / h]], device=device))
    return torch.cat(masks, 1), torch.stack(ratios, 1)


def _shapes(hw, device):
    t = torch.tensor(hw, dtype=torch.long, device=device)
    t._hw_list = list(hw)
    return t


def test_deformable_encoder_layer_train_mode_matches_fp64(cuda_device, strict_fp32, monkeypatch):
    from trackformer_b200.deformable_transformer import DeformableTransformerEncoder, DeformableTransformerEncoderLayer
    torch.manual_seed(0)
    layer = DeformableTransformerEncoderLayer(256, 1024, P_DROP, "relu", 4, 8, 4).to(cuda_device)
    _perturb_(layer, 1)
    layer.train()
    B, S = 2, sum(h * w for h, w in C2_HW)
    pad, ratios = _level_padding(C2_HW, B, cuda_device)
    shapes = _shapes(C2_HW, cuda_device)
    ref_pts = DeformableTransformerEncoder.get_reference_points(shapes, ratios, cuda_device)
    g = torch.Generator().manual_seed(2)
    src = torch.randn(B, S, 256, generator=g).to(cuda_device).requires_grad_(True)
    pos = torch.randn(B, S, 256, generator=g).to(cuda_device)
    gout = torch.randn(B, S, 256, generator=g).to(cuda_device)
    rec = _Recorder(monkeypatch, layer)
    out = layer(src, pos, ref_pts, shapes, pad)
    out.backward(gout)
    rp = rec.replay()
    assert rp.n_seeds == 3
    P = _params64(layer)
    src64 = src.detach().double().requires_grad_(True)
    ref_out = _deformable_encoder_layer_ref(P, "", src64, pos.double(), ref_pts.double(), C2_HW, pad, rp, P_DROP)
    rp.done()
    ref_out.backward(gout.double())
    _compare_layer(layer, P, {"src": src}, {"src": src64}, out, ref_out, 1e-3, 1e-4, 1e-3,
                   loose=("sampling_offsets", "attention_weights"), kinked=("src",))


def test_deformable_decoder_layer_train_mode_matches_fp64(cuda_device, strict_fp32, monkeypatch):
    """300 object queries after 40 track-query slots, the tail of each image's track slots filler (hidden as keys, as
    GraphedDetector pads them), into C2 memory of a padded batch of two."""
    from trackformer_b200.deformable_transformer import DeformableTransformerDecoderLayer
    torch.manual_seed(0)
    layer = DeformableTransformerDecoderLayer(256, 1024, P_DROP, "relu", 4, 8, 4).to(cuda_device)
    _perturb_(layer, 3)
    layer.train()
    B, S, T, Q = 2, sum(h * w for h, w in C2_HW), 40, 300
    Lq = T + Q
    pad, ratios = _level_padding(C2_HW, B, cuda_device)
    shapes = _shapes(C2_HW, cuda_device)
    filler = torch.zeros(B, Lq, dtype=torch.bool, device=cuda_device)
    filler[0, 31:T] = True
    filler[1, 17:T] = True
    g = torch.Generator().manual_seed(4)
    tgt = torch.randn(B, Lq, 256, generator=g).to(cuda_device).requires_grad_(True)
    qpos = torch.randn(B, Lq, 256, generator=g)
    qpos[:, :T] = 0.0                                                    # track queries carry no positional part
    qpos = qpos.to(cuda_device)
    memory = torch.randn(B, S, 256, generator=g).to(cuda_device).requires_grad_(True)
    boxes = torch.cat([torch.rand(B, Lq, 2, generator=g) * 0.6 + 0.2, torch.rand(B, Lq, 2, generator=g) * 0.25 + 0.05], -1)
    ref_in = (boxes.to(cuda_device)[:, :, None] * torch.cat([ratios, ratios], -1)[:, None]).contiguous()
    gout = torch.randn(B, Lq, 256, generator=g).to(cuda_device)
    rec = _Recorder(monkeypatch, layer)
    out = layer(tgt, qpos, ref_in, memory, shapes, pad, None, filler)
    out.backward(gout)
    rp = rec.replay()
    assert rp.n_seeds == 4 and set(rp.stock) == {"dropout3"}
    P = _params64(layer)
    tgt64, mem64 = (t.detach().double().requires_grad_(True) for t in (tgt, memory))
    ref_out = _deformable_decoder_layer_ref(P, "", tgt64, qpos.double(), ref_in.double(), mem64, C2_HW, pad, filler, rp,
                                            P_DROP)
    rp.done()
    ref_out.backward(gout.double())
    _compare_layer(layer, P, {"tgt": tgt, "memory": memory}, {"tgt": tgt64, "memory": mem64}, out, ref_out, 1e-3, 1e-4,
                   1e-3, loose=("sampling_offsets", "attention_weights"), kinked=("tgt",))


@pytest.mark.parametrize("pre_norm", [False, True], ids=["post_norm", "pre_norm"])
def test_vanilla_encoder_layer_train_mode_matches_fp64(cuda_device, strict_fp32, monkeypatch, pre_norm):
    from trackformer_b200.transformer import TransformerEncoderLayer
    torch.manual_seed(0)
    layer = TransformerEncoderLayer(256, 8, 2048, P_DROP, "relu", pre_norm).to(cuda_device)
    _perturb_(layer, 5)
    layer.train()
    B, L = 2, 1050
    pad = _image_padding(B, (25, 42), [(25, 42), (18, 37)], cuda_device)
    g = torch.Generator().manual_seed(6)
    src = torch.randn(L, B, 256, generator=g).to(cuda_device).requires_grad_(True)
    pos = torch.randn(L, B, 256, generator=g).to(cuda_device)
    gout = torch.randn(L, B, 256, generator=g).to(cuda_device)
    rec = _Recorder(monkeypatch, layer)
    out = layer(src, src_key_padding_mask=pad, pos=pos)
    out.backward(gout)
    rp = rec.replay()
    assert rp.n_seeds == (2 if pre_norm else 4)
    P = _params64(layer)
    src64 = src.detach().double().requires_grad_(True)
    ref_out = _encoder_layer_ref(P, "", src64, pad, pos.double(), pre_norm, rp, P_DROP)
    rp.done()
    ref_out.backward(gout.double())
    _compare_layer(layer, P, {"src": src}, {"src": src64}, out, ref_out, 1e-4, 1e-5, 1e-4)


@pytest.mark.parametrize("pre_norm", [False, True], ids=["post_norm", "pre_norm"])
def test_vanilla_decoder_layer_train_mode_matches_fp64(cuda_device, strict_fp32, monkeypatch, pre_norm):
    """100 object queries + 20 track queries (the last 6 of the second image filler) into 1050 padded memory tokens."""
    from trackformer_b200.transformer import TransformerDecoderLayer
    torch.manual_seed(0)
    layer = TransformerDecoderLayer(256, 8, 2048, P_DROP, "relu", pre_norm).to(cuda_device)
    _perturb_(layer, 7)
    layer.train()
    B, Q, T, L = 2, 100, 20, 1050
    mem_pad = _image_padding(B, (25, 42), [(25, 42), (21, 30)], cuda_device)
    tgt_pad = torch.zeros(B, Q + T, dtype=torch.bool, device=cuda_device)
    tgt_pad[1, Q + T - 6:] = True
    g = torch.Generator().manual_seed(8)
    tgt = torch.randn(Q + T, B, 256, generator=g).to(cuda_device).requires_grad_(True)
    qpos = torch.randn(Q + T, B, 256, generator=g)
    qpos[Q:] = 0.0
    qpos = qpos.to(cuda_device)
    memory = torch.randn(L, B, 256, generator=g).to(cuda_device).requires_grad_(True)
    pos = torch.randn(L, B, 256, generator=g).to(cuda_device)
    gout = torch.randn(Q + T, B, 256, generator=g).to(cuda_device)
    rec = _Recorder(monkeypatch, layer)
    out = layer(tgt, memory, tgt_key_padding_mask=tgt_pad, memory_key_padding_mask=mem_pad, pos=pos, query_pos=qpos)
    out.backward(gout)
    rp = rec.replay()
    assert rp.n_seeds == (3 if pre_norm else 6)
    P = _params64(layer)
    tgt64, mem64 = (t.detach().double().requires_grad_(True) for t in (tgt, memory))
    ref_out = _decoder_layer_ref(P, "", tgt64, mem64, tgt_pad, mem_pad, pos.double(), qpos.double(), pre_norm, rp, P_DROP)
    rp.done()
    ref_out.backward(gout.double())
    _compare_layer(layer, P, {"tgt": tgt, "memory": memory}, {"tgt": tgt64, "memory": mem64}, out, ref_out, 1e-4, 1e-5,
                   1e-4)


@pytest.mark.parametrize("pre_norm", [False, True], ids=["post_norm", "pre_norm"])
def test_vanilla_transformer_train_mode_matches_fp64(cuda_device, strict_fp32, monkeypatch, pre_norm):
    """The layers composed into Transformer (tests/transformer_fixtures.py geometry: two padded feature maps, 28
    queries of which 4 are track queries), one begin_step pool per pass."""
    import transformer_fixtures as tf
    from trackformer_b200.transformer import Transformer
    model = tf.build(Transformer, pre_norm).to(cuda_device).train()
    x = tf.inputs(cuda_device)
    tgt = x["tgt"].clone().requires_grad_(True)
    rec = _Recorder(monkeypatch, model)
    hs, _, memory = model(x["src"], x["mask"], x["query_embed"], x["pos"], tgt=tgt)
    (hs * x["weight"]).sum().backward()
    rp = rec.replay()
    P = _params64(model)
    tgt64 = tgt.detach().double().requires_grad_(True)
    B, C, h, w = x["src"].shape
    src = x["src"].double().flatten(2).permute(2, 0, 1)
    pos = x["pos"].double().flatten(2).permute(2, 0, 1)
    mask = x["mask"].flatten(1)
    qpos = x["query_embed"].double()
    mem = src
    for i in range(2):
        mem = _encoder_layer_ref(P, f"encoder.layers.{i}.", mem, mask, pos, pre_norm, rp, P_DROP)
    if pre_norm:
        mem = _ln(P, "encoder.norm.", mem)
    out, inter = tgt64, []
    for i in range(2):
        out = _decoder_layer_ref(P, f"decoder.layers.{i}.", out, mem, None, mask, pos, qpos, pre_norm, rp, P_DROP)
        inter.append(out)
    hs_ref = _ln(P, "decoder.norm.", torch.stack(inter)).transpose(1, 2)
    mem_ref = mem.permute(1, 2, 0).reshape(B, C, h, w)
    rp.done()
    (hs_ref * x["weight"].double()).sum().backward()
    _close("hs", hs.detach(), hs_ref.detach(), 1e-4, 1e-5)
    _close("memory", memory.detach(), mem_ref.detach(), 1e-4, 1e-5)
    _close("grad tgt", tgt.grad, tgt64.grad, 1e-4, 1e-5)
    params = dict(model.named_parameters())
    for k in tf.GRAD_KEYS:
        _close(f"grad {k}", params[k].grad, P[k].grad, 1e-3, 1e-4)


# ------------------------------------------------------------------------------------------------------------------
# 5. seeds and CUDA graphs
# ------------------------------------------------------------------------------------------------------------------
def _pool_draws(monkeypatch, model, run):
    from trackformer_b200 import seeds
    rec = _Recorder(monkeypatch, model)
    run()
    rec.replay()
    values = [int(s.item()) for s in rec.drawn]
    assert seeds._pool is not None and seeds._next == len(values), "a fused site drew its seed outside the pool"
    return values, rec.stock


def test_one_seed_per_fused_site_deformable(cuda_device, monkeypatch):
    """Six encoder layers x (norm1, FFN ReLU, norm2) + six decoder layers x (self-attention, norm2, norm1, norm3) = 42;
    the decoder FFN's dropout3 is the stock module."""
    from trackformer_b200 import seeds
    from trackformer_b200.deformable_transformer import DeformableTransformer
    torch.manual_seed(0)
    model = DeformableTransformer(256, 8, 6, 6, 1024, P_DROP, return_intermediate_dec=True).to(cuda_device).train()
    hw = [(24, 32), (12, 16), (6, 8), (3, 4)]
    g = torch.Generator().manual_seed(0)
    srcs = [torch.randn(2, 256, h, w, generator=g).to(cuda_device) for h, w in hw]
    masks = [torch.zeros(2, h, w, dtype=torch.bool, device=cuda_device) for h, w in hw]
    pos = [torch.randn(2, 256, h, w, generator=g).to(cuda_device) for h, w in hw]
    query = torch.randn(300, 512, generator=g).to(cuda_device)
    values, stock = _pool_draws(monkeypatch, model, lambda: model(srcs, masks, pos, query))
    assert len(values) == 42 <= seeds._POOL_SIZE
    assert len(set(values)) == len(values)
    assert set(stock) == {f"decoder.layers.{i}.dropout3" for i in range(6)}


def test_one_seed_per_fused_site_vanilla(cuda_device, monkeypatch):
    """Six encoder layers x (attention, norm1, FFN ReLU, norm2) + six decoder layers x (self-attention, norm1,
    cross-attention, norm2, FFN ReLU, norm3) = 60, and no stock dropout module runs."""
    from trackformer_b200 import seeds
    from trackformer_b200.transformer import Transformer
    torch.manual_seed(0)
    model = Transformer(256, 8, 6, 6, 2048, P_DROP, return_intermediate_dec=True).to(cuda_device).train()
    g = torch.Generator().manual_seed(0)
    src = torch.randn(2, 256, 25, 42, generator=g).to(cuda_device)
    pos = torch.randn(2, 256, 25, 42, generator=g).to(cuda_device)
    mask = _image_padding(2, (25, 42), [(25, 42), (19, 33)], cuda_device).view(2, 25, 42)
    query = torch.randn(100, 2, 256, generator=g).to(cuda_device)
    values, stock = _pool_draws(monkeypatch, model, lambda: model(src, mask, query, pos))
    assert len(values) == 60 <= seeds._POOL_SIZE
    assert len(set(values)) == len(values)
    assert not stock


def _deterministic_begin_step(device):
    """seeds.begin_step with a fixed pool: still one captured device kernel (arange + multiply) per pass, so every replay
    rewrites the same seeds."""
    from trackformer_b200 import seeds
    idx = torch.arange(1, seeds._POOL_SIZE + 1, dtype=torch.int64, device=device)
    seeds._pool = idx * 0x5DEECE66D + 0xB
    seeds._next = 0


def test_graphed_train_step_equals_eager_with_dropout(cuda_device, strict_fp32, monkeypatch):
    """Vanilla DETR detection at dropout 0.1: under the same seeds the graphed step gives the eager step's loss and
    gradient (tolerances of the dropout-0 comparison in test_detr_gpu.py); every dropout site is a fused one."""
    import detr_fixtures as df
    from trackformer_b200 import seeds
    from trackformer_b200.train_step import TrainStep
    torch.manual_seed(0)
    model, criterion = df.build(False, False, device=str(cuda_device), enc_layers=2, dec_layers=3, dropout=P_DROP)
    model, criterion = model.to(cuda_device).train(), criterion.to(cuda_device).train()
    stock = []
    for name, m in model.named_modules():
        if isinstance(m, nn.Dropout):
            assert m.p == P_DROP
            m.register_forward_hook(lambda mod, inp, out, name=name: stock.append(name))
    model_e = copy.deepcopy(model)
    monkeypatch.setattr(seeds, "begin_step", _deterministic_begin_step)
    g = torch.Generator().manual_seed(3)
    frames = [torch.randn(1, 3, 192, 256, generator=g).to(cuda_device) for _ in range(3)]
    graphed = TrainStep(model, criterion, None, use_graphs=True, example_frames=frames[0])
    eager = TrainStep(model_e, criterion, None, use_graphs=False)
    for i, f in enumerate(frames):
        n = 4 + i
        gb = torch.Generator().manual_seed(10 + i)
        boxes = torch.cat([torch.rand(n, 2, generator=gb) * 0.5 + 0.25, torch.rand(n, 2, generator=gb) * 0.2 + 0.05], 1)
        tg = [{"boxes": boxes.to(cuda_device), "labels": torch.randint(0, 91, (n,), generator=gb).to(cuda_device)}]
        loss_g = graphed(f, tg).clone()
        loss_e = eager(f, tg)
        torch.testing.assert_close(loss_g, loss_e, rtol=1e-4, atol=1e-4)
        scale = float(eager.flat_grad.abs().max())
        torch.testing.assert_close(graphed.flat_grad, eager.flat_grad, rtol=1e-3, atol=2e-4 * scale)
    assert not stock, f"stock dropout modules ran: {sorted(set(stock))}"


def test_graph_replays_draw_fresh_masks(cuda_device, strict_fp32):
    """With the real pool, two replays on identical inputs give different losses and gradients: each replay draws new
    seeds (a pool baked in at capture would repeat the masks)."""
    import detr_fixtures as df
    from trackformer_b200.train_step import TrainStep
    torch.manual_seed(0)
    model, criterion = df.build(False, False, device=str(cuda_device), enc_layers=2, dec_layers=3, dropout=P_DROP)
    model, criterion = model.to(cuda_device).train(), criterion.to(cuda_device).train()
    g = torch.Generator().manual_seed(3)
    frame = torch.randn(1, 3, 192, 256, generator=g).to(cuda_device)
    graphed = TrainStep(model, criterion, None, use_graphs=True, example_frames=frame)
    boxes = torch.tensor([[0.3, 0.4, 0.1, 0.2], [0.6, 0.5, 0.2, 0.1], [0.5, 0.7, 0.15, 0.1]])
    tg = [{"boxes": boxes.to(cuda_device), "labels": torch.tensor([1, 5, 7]).to(cuda_device)}]
    losses, grads = [], []
    for _ in range(2):
        losses.append(float(graphed(frame, tg)))
        grads.append(graphed.flat_grad.clone())
    assert math.isfinite(losses[0]) and math.isfinite(losses[1])
    assert losses[0] != losses[1]
    assert not torch.equal(grads[0], grads[1])
