"""The vanilla transformer on the H100 kernels (dense attention for the encoder self-attention and the decoder
cross-attention, small attention for the decoder's query self-attention, fused FFN and residual norms) against the
reference's own ``Transformer`` recorded in tests/golden/transformer_{post,pre}.npz, in strict fp32 and with TF32
Linears; filler-query padding; and a training pass with dropout on the fused kernels."""
import numpy as np
import pytest
import torch

import transformer_fixtures as tf
from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture
def matmul_tf32(request):
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = request.param
    yield request.param
    torch.backends.cuda.matmul.allow_tf32 = old


def _check(res, gold, rtol, rel_atol):
    for k, g in gold.items():
        if k == "state_dict_shapes":
            continue
        scale = float(np.abs(g).max()) or 1.0
        np.testing.assert_allclose(res[k], g, rtol=rtol, atol=rel_atol * scale, err_msg=k)


@pytest.mark.parametrize("mode", ["post", "pre"])
@pytest.mark.parametrize("matmul_tf32", [False, True], ids=["fp32", "tf32"], indirect=True)
def test_matches_reference_fixture(cuda_device, mode, matmul_tf32):
    from trackformer_b200 import dense_attention
    from trackformer_b200.transformer import Transformer
    model = tf.build(Transformer, mode == "pre")
    assert dense_attention.supported(model.encoder.layers[0].self_attn, torch.zeros(1, device=cuda_device))
    gold = load_golden(mode, prefix="transformer_")
    res = tf.run_transformer(Transformer, mode == "pre", device=cuda_device)
    if matmul_tf32:
        # the library's TF32 Linears (10-bit mantissa, K up to 2048) move the raw hidden states by up to ~1 % of
        # their largest magnitude; the attention kernels themselves are fp32-accurate (the strict case above)
        for k in ("hs", "hs_without_norm_last", "memory"):
            scale = float(np.abs(gold[k]).max())
            assert float(np.abs(res[k] - gold[k]).max()) < 2e-2 * scale, k
    else:
        _check(res, gold, rtol=2e-4, rel_atol=2e-5)


def test_filler_queries_do_not_change_real_rows(cuda_device):
    from trackformer_b200.transformer import Transformer
    model = tf.build(Transformer, False).to(cuda_device)
    x = tf.inputs(cuda_device)
    n_fill = 9
    g = torch.Generator().manual_seed(3)
    fill = torch.randn(n_fill, 2, tf.D, generator=g).to(cuda_device)
    with torch.no_grad():
        ref = model(x["src"], x["mask"], x["query_embed"], x["pos"], tgt=x["tgt"])
        pad = torch.zeros(2, n_fill + tf.N_QUERIES, dtype=torch.bool, device=cuda_device)
        pad[:, :n_fill] = True
        got = model(x["src"], x["mask"], torch.cat([torch.zeros_like(fill), x["query_embed"]]), x["pos"],
                    tgt=torch.cat([fill, x["tgt"]]), tgt_key_padding_mask=pad)
    torch.testing.assert_close(got[0][:, :, n_fill:], ref[0], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(got[2], ref[2])


def test_training_pass_with_dropout(cuda_device):
    """Training mode: dropout on every fused site; the pass is finite, differs from eval, and has gradients everywhere."""
    from trackformer_b200.transformer import Transformer
    model = tf.build(Transformer, False).to(cuda_device)
    x = tf.inputs(cuda_device)
    with torch.no_grad():
        ev = model(x["src"], x["mask"], x["query_embed"], x["pos"], tgt=x["tgt"])[0]
    model.train()
    hs = model(x["src"], x["mask"], x["query_embed"], x["pos"], tgt=x["tgt"])[0]
    (hs * x["weight"]).sum().backward()
    assert torch.isfinite(hs).all() and not torch.allclose(hs, ev)
    for name, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
