"""ORACLE -- TEST INFRASTRUCTURE ONLY.  ctypes front-end of oracle/_ref/libmsda_refcuda.so: the reference's OWN CUDA
kernels (ms_deform_im2col_cuda.cuh) compiled for sm_90a from the reference sources (oracle/Makefile `ref`,
only where those sources are present).  GPU-vs-GPU parity checks and the "kernel to beat" timing use it; the product never does."""
from __future__ import annotations

import ctypes
import os

import torch

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libmsda_refcuda.so")
_lib = None


def available() -> bool:
    return os.path.exists(_SO)


def _load():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(_SO)
        vp, i = ctypes.c_void_p, ctypes.c_int
        _lib.refcuda_ws_bytes.restype = ctypes.c_int64
        _lib.refcuda_ws_bytes.argtypes = [i] * 7
        _lib.refcuda_forward_f32.argtypes = [vp] * 6 + [i] * 7 + [vp]
        _lib.refcuda_backward_f32.argtypes = [vp] * 9 + [i] * 7 + [vp]
    return _lib


def _dims(value, loc):
    n, s, m, d = value.shape
    _, lq, _, l, p, _ = loc.shape
    return n, s, m, d, l, lq, p


def forward(value, shapes, loc, attn, ws=None):
    lib = _load()
    n, s, m, d, l, lq, p = _dims(value, loc)
    if ws is None:
        ws = torch.empty(lib.refcuda_ws_bytes(n, m, d, l, lq, p, 4), dtype=torch.uint8, device=value.device)
    out = torch.empty(n, lq, m * d, device=value.device)
    rc = lib.refcuda_forward_f32(value.data_ptr(), shapes.data_ptr(), loc.data_ptr(), attn.data_ptr(), out.data_ptr(),
                                 ws.data_ptr(), n, s, m, d, l, lq, p, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return out


def backward(value, shapes, loc, attn, grad_out, ws=None):
    lib = _load()
    n, s, m, d, l, lq, p = _dims(value, loc)
    if ws is None:
        ws = torch.empty(l * 8 + 64, dtype=torch.uint8, device=value.device)
    gv, gl, ga = torch.empty_like(value), torch.empty_like(loc), torch.empty_like(attn)
    rc = lib.refcuda_backward_f32(value.data_ptr(), shapes.data_ptr(), loc.data_ptr(), attn.data_ptr(),
                                  grad_out.data_ptr(), gv.data_ptr(), gl.data_ptr(), ga.data_ptr(), ws.data_ptr(),
                                  n, s, m, d, l, lq, p, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return gv, gl, ga
