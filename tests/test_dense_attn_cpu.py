"""CPU side of the dense-attention path (csrc/dense_attn.cu): the C ABI rejects bad arguments without touching a GPU,
and the nn.MultiheadAttention replacement keeps the stock module where the kernels do not apply."""
import ctypes

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from trackformer_b200 import _build
    return ctypes.CDLL(_build.build_library())


def test_argument_validation_without_gpu(lib):
    f = lib.tfb200_dense_attn_fwd_f32
    f.restype = ctypes.c_int
    vp, i, fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    f.argtypes = [vp] * 7 + [i] * 4 + [vp, fl, fl, vp]
    buf = ctypes.create_string_buffer(256)
    base = (ctypes.addressof(buf) + 15) & ~15
    p = ctypes.c_void_p(base)
    strides = (ctypes.c_int64 * 8)(512, 256, 512, 256, 512, 256, 512, 256)
    s = ctypes.cast(strides, vp)
    assert f(None, p, p, None, None, p, p, 2, 8, 4, 4, s, 0.17, 1.0, None) == -1      # NULL q
    assert f(p, p, p, None, None, p, p, 2, 8, 0, 4, s, 0.17, 1.0, None) == -2         # Lq = 0
    assert f(p, p, p, None, None, p, p, 2, 8, 4, 0, s, 0.17, 1.0, None) == -2         # Lk = 0
    assert f(p, p, p, None, None, p, p, 2, 8, 4, 4, s, 0.17, 0.0, None) == -2         # keep_prob = 0
    odd = ctypes.c_void_p(base + 4)
    assert f(p, odd, p, None, None, p, p, 2, 8, 4, 4, s, 0.17, 1.0, None) == -2       # k not 16-byte aligned
    strides[2] = 514
    assert f(p, p, p, None, None, p, p, 2, 8, 4, 4, s, 0.17, 1.0, None) == -2         # k rows not 16-byte aligned
    b = lib.tfb200_dense_attn_bwd_f32
    b.restype = ctypes.c_int
    b.argtypes = [vp] * 12 + [i] * 4 + [vp, fl, fl, vp]
    assert b(*([p] * 11), None, 2, 8, 4, 4, s, 0.17, 1.0, None) == -1                # NULL delta workspace


def test_cpu_tensors_use_the_stock_module():
    from trackformer_b200 import dense_attention
    torch.manual_seed(0)
    mha = torch.nn.MultiheadAttention(256, 8, dropout=0.0).eval()
    q = torch.randn(7, 2, 256)
    mem = torch.randn(11, 2, 256)
    pad = torch.zeros(2, 11, dtype=torch.bool)
    pad[1, 6:] = True
    assert not dense_attention.supported(mha, q)
    got = dense_attention.attention(mha, q, mem, mem, pad)
    want = mha(q, mem, mem, key_padding_mask=pad)[0]
    torch.testing.assert_close(got, want)


def test_unsupported_head_width_is_reported():
    from trackformer_b200 import dense_attention
    mha = torch.nn.MultiheadAttention(256, 4)        # 64 channels per head
    q = torch.randn(3, 1, 256)
    assert not dense_attention.supported(mha, q)
