"""The host restatement of the fused kernels' dropout hash (tests/dropout_hash.py) on its own: the vectorised torch
arithmetic against a plain Python-integer statement, keep rates, the dependence on both halves of the seed and on both
halves of the element index, and the threshold's rounding and saturation."""
import numpy as np
import pytest
import torch

import dropout_hash as dh

SEEDS = [0, 1, 123456789012345, 2 ** 62 - 1, 0x0123456789ABCDEF]


@pytest.mark.parametrize("seed", SEEDS)
def test_vectorised_hash_equals_python_integers(seed):
    idx = [0, 1, 2, 31, 32, 1023, 22223 * 256 - 1, 2 ** 31, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 7, 3 * 2 ** 40 + 5]
    got = dh.hash32(seed, torch.tensor(idx, dtype=torch.int64)).tolist()
    assert got == [dh.hash32_scalar(seed, i) for i in idx]
    assert all(0 <= h <= dh.M32 for h in got)


def test_mix32_known_values():
    """mix32 is a bijection of uint32 with a fixed point at 0; pinned values guard the constants and the shifts."""
    x = torch.tensor([0, 1, 2, 0xFFFFFFFF, 0x9E3779B9], dtype=torch.int64)
    got = dh.mix32(x).tolist()
    want = []
    for v in x.tolist():
        v ^= v >> 16
        v = (v * 0x7FEB352D) % 2 ** 32
        v ^= v >> 15
        v = (v * 0x846CA68B) % 2 ** 32
        want.append(v ^ (v >> 16))
    assert got == want and got[0] == 0
    y = torch.arange(0, 1 << 20, dtype=torch.int64)
    assert torch.unique(dh.mix32(y)).numel() == y.numel()


@pytest.mark.parametrize("p", [0.1, 0.3, 0.5])
@pytest.mark.parametrize("seed", [7, 2 ** 40 + 3, 0x3FFFFFFFFFFFFFFF])
def test_keep_rate_within_four_sigma(seed, p):
    n = 1 << 20
    keep = 1.0 - p
    rate = float(dh.keep_mask(seed, n, keep).double().mean())
    sigma = (keep * p / n) ** 0.5
    assert abs(rate - keep) < 4 * sigma, (rate, keep, sigma)


def test_seeds_differing_in_one_half_give_different_masks():
    n = 1 << 16
    base = 0x0000123400005678
    ref = dh.keep_mask(base, n, 0.9)
    for other in (base ^ (1 << 40), base + (7 << 32), base ^ 1, base + 12345):
        m = dh.keep_mask(other, n, 0.9)
        diff = float((m != ref).double().mean())
        # two independent masks at keep 0.9 disagree on 2 * 0.9 * 0.1 = 18 % of the elements
        assert 0.16 < diff < 0.20, (hex(other), diff)


def test_high_index_word_enters_the_hash():
    """Elements 2^32 apart share their low index word: only hi32(idx) separates them."""
    n = 1 << 16
    lo = dh.keep_mask(99, n, 0.9)
    hi = dh.keep_mask(99, n, 0.9, offset=1 << 32)
    assert 0.16 < float((lo != hi).double().mean()) < 0.20


def test_threshold_rounds_through_fp32_and_saturates():
    assert dh.keep_threshold(1.0) == 0xFFFFFFFF
    assert dh.keep_threshold(1.0 - 1e-12) == 0xFFFFFFFF        # rounds to 1.0f
    assert dh.keep_threshold(0.5) == 1 << 31
    assert dh.keep_threshold(0.9) == int(float(np.float32(0.9)) * 2 ** 32) == 3865470464
    assert dh.keep_threshold(0.9) != int(0.9 * 2 ** 32)          # the double product would be 3865470566
    assert dh.keep_threshold(0.0) == 0
    # keep_prob = 1 keeps every element, whatever the hash
    assert bool(dh.keep_mask(5, 1 << 16, 1.0).all())


def test_site_shapes_are_views_of_the_flat_index():
    flat = dh.keep_mask(42, 2 * 8 * 33 * 77, 0.9)
    torch.testing.assert_close(dh.attention_mask(42, 2, 8, 33, 77, 0.9).flatten(), flat, rtol=0, atol=0)
    assert dh.layernorm_mask(42, 33, 128, 0.7).shape == (33, 128)
    assert torch.equal(dh.layernorm_mask(42, 33, 128, 0.7).flatten(), dh.keep_mask(42, 33 * 128, 0.7))
    assert dh.relu_dropout_mask(42, (2, 3, 4), 0.7).shape == (2, 3, 4)
