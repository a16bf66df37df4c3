"""The vanilla transformer (trackformer_b200/transformer.py) on CPU against the reference's own ``Transformer``, recorded
in tests/golden/transformer_{post,pre}.npz: outputs, gradients, state_dict names and shapes; plus the arguments it
rejects and the filler-query padding of the decoder's self-attention."""
import json
from argparse import Namespace

import numpy as np
import pytest
import torch

import transformer_fixtures as tf
from conftest import load_golden


def _check(res, gold, rtol=1e-4, rel_atol=1e-5):
    for k, g in gold.items():
        if k == "state_dict_shapes":
            continue
        scale = float(np.abs(g).max()) or 1.0
        np.testing.assert_allclose(res[k], g, rtol=rtol, atol=rel_atol * scale, err_msg=k)


@pytest.mark.parametrize("mode", ["post", "pre"])
def test_matches_reference_fixture(mode):
    from trackformer_b200.transformer import Transformer
    gold = load_golden(mode, prefix="transformer_")
    _check(tf.run_transformer(Transformer, mode == "pre"), gold)


@pytest.mark.parametrize("mode", ["post", "pre"])
def test_state_dict_names_and_shapes_equal_the_reference(mode):
    from trackformer_b200.transformer import Transformer
    gold = load_golden(mode, prefix="transformer_")
    want = {k: tuple(v) for k, v in json.loads(str(gold["state_dict_shapes"])).items()}
    got = tf.state_dict_shapes(Transformer, mode == "pre")
    assert list(got) == list(want)
    assert got == want
    assert "decoder.layers.5.multihead_attn.in_proj_weight" in got and "decoder.norm.weight" in got


def _args(**kw):
    base = dict(hidden_dim=256, dropout=0.1, nheads=8, dim_feedforward=2048, enc_layers=6, dec_layers=6, pre_norm=False,
                track_attention=False)
    base.update(kw)
    return Namespace(**base)


def test_build_transformer_geometry():
    from trackformer_b200.transformer import build_transformer
    t = build_transformer(_args())
    assert t.d_model == 256 and t.nhead == 8 and t.decoder.return_intermediate
    assert len(t.encoder.layers) == 6 and len(t.decoder.layers) == 6 and t.encoder.norm is None
    assert build_transformer(_args(pre_norm=True)).encoder.norm is not None


def test_track_attention_is_rejected():
    from trackformer_b200.transformer import build_transformer
    with pytest.raises(NotImplementedError, match="track_attention"):
        build_transformer(_args(track_attention=True))


def test_filler_queries_do_not_change_real_rows():
    """Filler rows prepended to the queries and hidden as self-attention keys leave every real row as it was."""
    from trackformer_b200.transformer import Transformer
    model = tf.build(Transformer, False)
    x = tf.inputs()
    n_fill = 5
    g = torch.Generator().manual_seed(3)
    fill = torch.randn(n_fill, 2, tf.D, generator=g)
    with torch.no_grad():
        ref = model(x["src"], x["mask"], x["query_embed"], x["pos"], tgt=x["tgt"])
        pad = torch.zeros(2, n_fill + tf.N_QUERIES, dtype=torch.bool)
        pad[:, :n_fill] = True
        got = model(x["src"], x["mask"], torch.cat([torch.zeros_like(fill), x["query_embed"]]), x["pos"],
                    tgt=torch.cat([fill, x["tgt"]]), tgt_key_padding_mask=pad)
    torch.testing.assert_close(got[0][:, :, n_fill:], ref[0], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(got[2], ref[2])
