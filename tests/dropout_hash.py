"""Host restatement of the mask-free dropout of the fused kernels: which elements a given int64 seed keeps.

Every fused dropout site draws one int64 seed (trackformer_b200/seeds.py) and keeps element ``idx`` iff

    h    = mix32(lo32(idx) ^ mix32(hi32(idx) + lo32(seed)) ^ (hi32(seed) * 0x9e3779b9 mod 2^32))
    keep = h < keep_threshold(keep_prob)

which is restated here from the three copies of the hash:

    csrc/fused_norm.cu:37-44   mix32 / keep_elem          csrc/fused_norm.cu:358-361   keep_threshold
    csrc/small_attn.cu:27-34   mix32 / keep_elem          csrc/small_attn.cu:248-251   keep_threshold
    csrc/dense_attn.cu:37-44   mix32 / keep_elem          csrc/dense_attn.cu:421-424   keep_threshold

``idx`` is the logical element index of each site:

    fused LayerNorm   row * C + c (leading dims flattened into row)   fused_norm.cu:87-91 (forward), :189-193 (backward)
    relu_dropout      flat index of the contiguous input              fused_norm.cu:324-327
    attention         ((b * H + h) * Lq + q) * Lk + k                  small_attn.cu:102, 162, 230; dense_attn.cu:192, 301, 388

The arithmetic runs in torch int64 with explicit 32-bit masking (products split so that none overflows int64), on the
device of the caller's choice, so CPU tests check the restatement itself and GPU tests compare it with the kernels.
"""
from __future__ import annotations

import numpy as np
import torch

M32 = 0xFFFFFFFF
GOLDEN = 0x9E3779B9
_CHUNK = 1 << 24


def keep_threshold(keep_prob: float) -> int:
    """floor(keep_prob * 2^32) with keep_prob rounded to fp32 first (the kernels take it as a float), saturating at
    0xffffffff -- so keep_prob = 1 keeps every element."""
    t = float(np.float32(keep_prob)) * 4294967296.0
    return M32 if t >= 4294967295.0 else int(t)


def _mul32(x: torch.Tensor, c: int) -> torch.Tensor:
    """(x * c) mod 2^32 for x in [0, 2^32) and a 32-bit constant c, without int64 overflow."""
    lo, hi = c & 0xFFFF, c >> 16
    return (x * lo + (((x * hi) & 0xFFFF) << 16)) & M32


def mix32(x: torch.Tensor) -> torch.Tensor:
    """x ^= x >> 16; x *= 0x7feb352d; x ^= x >> 15; x *= 0x846ca68b; x ^= x >> 16   (uint32, held in int64)."""
    x = x & M32
    x = x ^ (x >> 16)
    x = _mul32(x, 0x7FEB352D)
    x = x ^ (x >> 15)
    x = _mul32(x, 0x846CA68B)
    return x ^ (x >> 16)


def hash32(seed: int, idx: torch.Tensor) -> torch.Tensor:
    """The 32-bit hash h of the elements ``idx`` (int64, >= 0) under ``seed``."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    s_lo, s_hi = seed & M32, seed >> 32
    salt = (s_hi * GOLDEN) & M32
    inner = mix32(((idx >> 32) + s_lo) & M32)
    return mix32((idx & M32) ^ inner ^ salt)


def keep_mask(seed: int, n_or_shape, keep_prob: float, device="cpu", offset: int = 0) -> torch.Tensor:
    """Bool keep mask of elements offset .. offset + n - 1, shaped like ``n_or_shape`` (an int or a shape)."""
    shape = (int(n_or_shape),) if isinstance(n_or_shape, (int, np.integer)) else tuple(int(s) for s in n_or_shape)
    n = int(np.prod(shape, dtype=np.int64)) if shape else 1
    th = keep_threshold(keep_prob)
    out = torch.empty(n, dtype=torch.bool, device=device)
    for a in range(0, n, _CHUNK):
        b = min(n, a + _CHUNK)
        idx = torch.arange(offset + a, offset + b, dtype=torch.int64, device=device)
        out[a:b] = hash32(seed, idx) < th
    return out.view(shape)


def layernorm_mask(seed: int, rows: int, C: int, keep_prob: float, device="cpu") -> torch.Tensor:
    """[rows, C] keep mask of the fused residual + dropout + LayerNorm (``x + dropout(branch)``)."""
    return keep_mask(seed, (rows, C), keep_prob, device)


def relu_dropout_mask(seed: int, shape, keep_prob: float, device="cpu") -> torch.Tensor:
    """Keep mask of ``relu_dropout`` in the shape of its (contiguous) input."""
    return keep_mask(seed, tuple(shape), keep_prob, device)


def attention_mask(seed: int, B: int, H: int, Lq: int, Lk: int, keep_prob: float, device="cpu") -> torch.Tensor:
    """[B, H, Lq, Lk] keep mask of the attention weights of the small- and dense-attention kernels."""
    return keep_mask(seed, (B, H, Lq, Lk), keep_prob, device)


def hash32_scalar(seed: int, idx: int) -> int:
    """The same hash on Python integers, one element (an independent statement for the CPU tests)."""
    def mix(x):
        x &= M32
        x ^= x >> 16
        x = (x * 0x7FEB352D) & M32
        x ^= x >> 15
        x = (x * 0x846CA68B) & M32
        return x ^ (x >> 16)
    seed &= 0xFFFFFFFFFFFFFFFF
    return mix((idx & M32) ^ mix((idx >> 32) + (seed & M32)) ^ (((seed >> 32) * GOLDEN) & M32))
