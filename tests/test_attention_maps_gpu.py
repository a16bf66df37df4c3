"""Head-averaged attention weights on the H100 (csrc/dense_attn.cu dense_attn_weights_kernel) against an fp64
restatement that forms its own softmax, ``attention(need_weights=True)`` against the stock nn.MultiheadAttention, and
Tracker (eager model, GraphedDetector replay, replay across padded-bucket boundaries) and DeviceTracker with
generate_attention_maps against the reference's tracker (tests/golden/make_golden_attention_maps.py) and each other."""
import numpy as np
import pytest
import torch

import attention_map_fixtures as amf
import detr_fixtures as df
from conftest import load_golden
from test_attention_maps_cpu import check_against_golden

pytestmark = pytest.mark.gpu


@pytest.fixture()
def strict_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _views(lq, lk, b, h, dev, seed):
    """q [Lq, B, H, 32] and k / v [Lk, B, H, 32] as strided views of packed projections, as the module passes them."""
    g = torch.Generator(device=dev).manual_seed(seed)
    e = 32 * h
    qp = torch.randn(lq, b, 2 * e, device=dev, generator=g)
    kv = torch.randn(lk, b, 3 * e, device=dev, generator=g)
    q = qp[..., :e].unflatten(-1, (h, 32))
    k = kv[..., e:2 * e].unflatten(-1, (h, 32))
    v = kv[..., 2 * e:].unflatten(-1, (h, 32))
    return q, k, v


def _reference(q, k, pad, scale):
    s = torch.einsum("qbhc,kbhc->bhqk", q.double(), k.double()) * scale
    if pad is not None:
        s = s.masked_fill(pad[:, None, None, :], float("-inf"))
    return torch.softmax(s, -1).mean(1)                               # [B, Lq, Lk]


@pytest.mark.parametrize("lq,lk", [(300, 1050), (400, 1050), (300, 1008), (400, 1008), (300, 4200), (400, 4200)])
def test_weights_kernel_matches_fp64(cuda_device, lq, lk):
    from trackformer_b200 import ext
    m = ext.load()
    q, k, v = _views(lq, lk, 1, 8, cuda_device, lq + lk)
    scale = 32 ** -0.5
    _, lse = m.dense_attention_forward(q, k, v, None, None, scale, 1.0)
    w = m.dense_attention_weights(q, k, None, lse, scale)
    assert w.shape == (1, lq, lk) and w.is_contiguous()
    ref = _reference(q, k, None, scale)
    torch.testing.assert_close(w.double(), ref, rtol=1e-4, atol=1e-7)
    torch.testing.assert_close(w.double().sum(-1), torch.ones(1, lq, dtype=torch.float64, device=cuda_device),
                               rtol=0, atol=1e-5)
    assert torch.equal(w, m.dense_attention_weights(q, k, None, lse, scale))       # no atomics: bitwise repeatable


def test_weights_kernel_padded_batch(cuda_device):
    from trackformer_b200 import ext
    m = ext.load()
    lq, lk = 333, 1050
    q, k, v = _views(lq, lk, 2, 8, cuda_device, 7)
    pad = torch.zeros(2, lk, dtype=torch.bool, device=cuda_device)
    pad[1, 613:] = True                                               # second image: padded keys
    pad[1, ::97] = True
    scale = 32 ** -0.5
    _, lse = m.dense_attention_forward(q, k, v, pad, None, scale, 1.0)
    w = m.dense_attention_weights(q, k, pad, lse, scale)
    ref = _reference(q, k, pad, scale)
    torch.testing.assert_close(w.double(), ref, rtol=1e-4, atol=1e-7)
    assert torch.count_nonzero(w[1][:, pad[1]]) == 0                  # exactly 0, not merely small
    assert torch.all(w[0] > 0)
    torch.testing.assert_close(w.double().sum(-1), torch.ones(2, lq, dtype=torch.float64, device=cuda_device),
                               rtol=0, atol=1e-5)
    assert torch.equal(w, m.dense_attention_weights(q, k, pad, lse, scale))


def test_attention_need_weights_matches_stock_module(cuda_device, strict_fp32):
    from trackformer_b200 import dense_attention
    torch.manual_seed(0)
    mha = torch.nn.MultiheadAttention(256, 8, dropout=0.1).to(cuda_device).eval()
    tgt = torch.randn(120, 2, 256, device=cuda_device)
    mem = torch.randn(1050, 2, 256, device=cuda_device)
    pos = torch.randn(1050, 2, 256, device=cuda_device)
    pad = torch.zeros(2, 1050, dtype=torch.bool, device=cuda_device)
    pad[1, 700:] = True
    assert dense_attention.supported(mha, tgt)
    with torch.no_grad():
        out, w = dense_attention.attention(mha, tgt, mem + pos, mem, pad, need_weights=True)
        want_out, want_w = mha(tgt, mem + pos, mem, key_padding_mask=pad, need_weights=True)
        plain = dense_attention.attention(mha, tgt, mem + pos, mem, pad)
    assert w.shape == want_w.shape == (2, 120, 1050)
    torch.testing.assert_close(w, want_w, rtol=1e-4, atol=1e-7)
    torch.testing.assert_close(out, want_out, rtol=1e-4, atol=1e-5)
    assert torch.equal(out, plain)                                    # asking for the weights leaves the output alone
    mha.train()
    with pytest.raises(NotImplementedError):
        dense_attention.attention(mha, tgt, mem + pos, mem, pad, need_weights=True)


def test_trackers_with_maps_match_reference_and_each_other(cuda_device, strict_fp32):
    """DETRSegmTracking with masks: Tracker over the eager model, over GraphedDetector replay, over replay with a
    bucket of 3 (track counts cross bucket boundaries), and DeviceTracker over replay."""
    from trackformer_b200.deformable_detr import PostProcess
    from trackformer_b200.device_tracker import DeviceTracker
    from trackformer_b200.graphed_detector import GraphedDetector
    from trackformer_b200.segmentation import PostProcessSegm
    from trackformer_b200.tracker import Tracker
    gold = load_golden("attention_maps_segm", "tracker_")

    def build(tracking, multi_frame, **kw):
        return df.build(tracking, multi_frame, device=str(cuda_device), **kw)
    arms = (("eager", Tracker, None), ("graph", Tracker, 16), ("padded", Tracker, 3), ("device", DeviceTracker, 16))
    outs = {}
    for name, cls, bucket in arms:
        wrap = None if bucket is None else (lambda mdl, b=bucket: GraphedDetector(mdl, bucket=b))
        outs[name] = amf.run_sequence(build, cls, {"bbox": PostProcess(), "segm": PostProcessSegm()},
                                      amf.golden_cfg(gold), gold["class_bias"], device=cuda_device, wrap=wrap)
        check_against_golden(outs[name], gold, map_atol=2e-5)
    a = outs["graph"]
    for other in ("eager", "padded", "device"):
        b = outs[other]
        np.testing.assert_array_equal(a["map_keys"], b["map_keys"], err_msg=other)
        np.testing.assert_allclose(a["maps"], b["maps"], rtol=1e-4, atol=1e-6, err_msg=other)
