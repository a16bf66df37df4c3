"""Autograd binding of the H100 MSDeformAttn kernels.

Mirror of the reference's ``MSDeformAttnFunction``
(src/trackformer/models/ops/functions/ms_deform_attn_func.py:14-31): same ``apply`` signature
``(value, value_spatial_shapes, sampling_locations, attention_weights, im2col_step)``, gradients for
arguments 0, 2 and 3 only, ``once_differentiable`` backward.  The compiled extension is resolved
through :mod:`trackformer_b200.ext` -- it must exist; there is no PyTorch fallback here (the
pure-PyTorch restatement lives in ``oracle/`` and is test infrastructure only).
"""
from __future__ import annotations

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ext

# Optional per-launch timing (bench.py's roofline leg): when a list is installed here, every forward /
# backward call is bracketed by CUDA events recorded on the launching stream and appended as
# (kind, (N, S, M, D, L, Lq, P), start_event, end_event).  None (default) = no events, no overhead.
_TIMING_SINK = None


def set_timing_sink(sink):
    """Install (or remove, with None) the list that receives per-launch CUDA-event records."""
    global _TIMING_SINK
    _TIMING_SINK = sink


def _dims(value, loc):
    n, s, m, d = value.shape
    _, lq, _, l, p, _ = loc.shape
    return (n, s, m, d, l, lq, p)


class MSDeformAttnFunction(Function):
    @staticmethod
    def forward(ctx, value, value_spatial_shapes, sampling_locations, attention_weights, im2col_step):
        msda = ext.load()
        ctx.im2col_step = int(im2col_step)
        sink = _TIMING_SINK
        if sink is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        out = msda.ms_deform_attn_forward(value, value_spatial_shapes, sampling_locations,
                                          attention_weights, ctx.im2col_step)
        if sink is not None:
            e1.record()
            sink.append(("fwd", _dims(value, sampling_locations), e0, e1))
        ctx.save_for_backward(value, value_spatial_shapes, sampling_locations, attention_weights)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        return _backward(ctx, grad_output, None)


def _backward(ctx, grad_output, hw):
    """Fused backward launch (grad_value, grad_sampling_loc, grad_attn_weight); ``hw`` (host level sizes) selects the
    encoder tile kernel."""
    value, shapes, loc, attn = ctx.saved_tensors
    sink = _TIMING_SINK
    if sink is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    if hw is None:
        g_value, g_loc, g_attn = ext.load().ms_deform_attn_backward(
            value, shapes, loc, attn, grad_output.contiguous(), ctx.im2col_step)
    else:
        g_value, g_loc, g_attn = ext.load().ms_deform_attn_backward_enc(
            value, shapes, loc, attn, grad_output.contiguous(), hw, ctx.im2col_step)
    if sink is not None:
        e1.record()
        sink.append(("bwd", _dims(value, loc), e0, e1))
    return g_value, None, g_loc, g_attn, None


# Which forward kernel serves an encoder call (queries == pixels): "tile" = the TMA-staged tile kernel
# (csrc/msda_enc_tma.cuh), "direct" = the 8-lane-group kernel.  Which one is faster depends on how compact the sampling
# pattern of neighbouring queries is (the tile kernel wins on the grid pattern of a freshly initialised model and loses
# once the locations scatter), so in "auto"
# mode the first eager call of a geometry times both on the data at hand and the winner is kept for that geometry.
import os as _os

_TILED_ENC = _os.environ.get("TFB200_TILED_ENC", "auto")            # "auto" | "1" (always tile) | "0" (never)
_TILED_ENC_BWD = _os.environ.get("TFB200_TILED_ENC_BWD", "auto")     # the same three modes for the backward tile kernel
_ENC_CHOICE = {}
_ENC_BWD_CHOICE = {}


def _time_us(fn, iters=3):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def encoder_kernel_choice(msda, value, shapes, loc, attn, hw, step):
    if _TILED_ENC in ("0", "1"):
        return "tile" if _TILED_ENC == "1" else "direct"
    key = (tuple(value.shape), tuple(hw), value.device.index)
    choice = _ENC_CHOICE.get(key)
    if choice is None:
        if torch.cuda.is_current_stream_capturing():
            return "direct"                                          # no timing inside a capture; decided by an eager call
        t_tile = _time_us(lambda: msda.ms_deform_attn_forward_enc(value, shapes, loc, attn, hw, step))
        t_direct = _time_us(lambda: msda.ms_deform_attn_forward(value, shapes, loc, attn, step))
        choice = _ENC_CHOICE[key] = "tile" if t_tile < 0.97 * t_direct else "direct"
    return choice


def encoder_backward_choice(msda, value, shapes, loc, attn, grad_out, hw, step):
    """Same one-time measurement for the backward."""
    if _TILED_ENC_BWD in ("0", "1"):
        return "tile" if _TILED_ENC_BWD == "1" else "direct"
    key = (tuple(value.shape), tuple(hw), value.device.index)
    choice = _ENC_BWD_CHOICE.get(key)
    if choice is None:
        if torch.cuda.is_current_stream_capturing():
            return "direct"
        t_tile = _time_us(lambda: msda.ms_deform_attn_backward_enc(value, shapes, loc, attn, grad_out, hw, step))
        t_direct = _time_us(lambda: msda.ms_deform_attn_backward(value, shapes, loc, attn, grad_out, step))
        choice = _ENC_BWD_CHOICE[key] = "tile" if t_tile < 0.97 * t_direct else "direct"
    return choice


class MSDeformAttnEncFunction(Function):
    """Encoder self-attention variant (queries are the pixels, ``Lq == S``): the forward may run the TMA-staged tile
    kernel, which needs the level sizes on the host -- taken from the ``_hw_list`` the transformer attaches to
    ``value_spatial_shapes``.  Results are those of :class:`MSDeformAttnFunction`; geometries the tile kernel does not
    cover fall through to the general kernel inside the extension (still CUDA -- there is no CPU path)."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, sampling_locations, attention_weights, im2col_step):
        msda = ext.load()
        ctx.im2col_step = int(im2col_step)
        hw = [int(v) for pair in value_spatial_shapes._hw_list for v in pair]
        ctx.hw = hw
        tile = encoder_kernel_choice(msda, value, value_spatial_shapes, sampling_locations, attention_weights, hw,
                                     ctx.im2col_step) == "tile"
        sink = _TIMING_SINK
        if sink is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        if tile:
            out = msda.ms_deform_attn_forward_enc(value, value_spatial_shapes, sampling_locations, attention_weights,
                                                  hw, ctx.im2col_step)
        else:
            out = msda.ms_deform_attn_forward(value, value_spatial_shapes, sampling_locations, attention_weights,
                                              ctx.im2col_step)
        if sink is not None:
            e1.record()
            sink.append(("fwd", _dims(value, sampling_locations), e0, e1))
        ctx.save_for_backward(value, value_spatial_shapes, sampling_locations, attention_weights)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, shapes, loc, attn = ctx.saved_tensors
        tile = encoder_backward_choice(ext.load(), value, shapes, loc, attn, grad_output.contiguous(), ctx.hw,
                                       ctx.im2col_step) == "tile"
        return _backward(ctx, grad_output, ctx.hw if tile else None)


class MSDeformAttnEncFusedFunction(Function):
    """Encoder tile kernels with the module's location / softmax arithmetic inside (SURVEY 8(f1): sampling locations and
    attention weights are never materialised): ``proj`` is the raw output of the [sampling_offsets | attention_weights]
    projections, ``reference_points`` [N, Lq, 4, 2], ``hw`` the host level sizes.  Gradients for ``value`` and ``proj``.
    bench.py's roofline leg keeps the UNFUSED algorithmic bytes as the yardstick for these launches."""

    @staticmethod
    def forward(ctx, value, proj, reference_points, hw):
        msda = ext.load()
        ctx.hw = list(hw)
        sink = _TIMING_SINK
        if sink is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        out = msda.ms_deform_attn_forward_enc_fused(value, proj, reference_points, ctx.hw)
        if sink is not None:
            e1.record()
            n, s_, m, d = value.shape
            sink.append(("fwd", (n, s_, m, d, 4, proj.shape[1], 4), e0, e1))
        ctx.save_for_backward(value, proj, reference_points)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, proj, ref = ctx.saved_tensors
        sink = _TIMING_SINK
        if sink is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        gv, gp = ext.load().ms_deform_attn_backward_enc_fused(value, proj, ref, grad_output.contiguous(), ctx.hw)
        if sink is not None:
            e1.record()
            n, s_, m, d = value.shape
            sink.append(("bwd", (n, s_, m, d, 4, proj.shape[1], 4), e0, e1))
        return gv, gp, None, None


_ENC_FUSED_CHOICE = {}
_TILED_ENC_FUSED = _os.environ.get("TFB200_TILED_ENC_FUSED", "auto")     # "auto" | "1" | "0"


def encoder_fused_choice(key, time_fused, time_unfused) -> bool:
    """One-time decision per geometry between the fused-prologue tile kernels and the materialising path (sampling-prep
    kernel + the autotuned op); both callables run the complete forward alternative once and are timed on the data at hand."""
    if _TILED_ENC_FUSED in ("0", "1"):
        return _TILED_ENC_FUSED == "1"
    choice = _ENC_FUSED_CHOICE.get(key)
    if choice is None:
        if torch.cuda.is_current_stream_capturing():
            return False
        choice = _ENC_FUSED_CHOICE[key] = _time_us(time_fused) < 0.97 * _time_us(time_unfused)
    return choice


def ms_deform_attn(value: torch.Tensor, spatial_shapes: torch.Tensor, sampling_locations: torch.Tensor,
                   attention_weights: torch.Tensor, im2col_step: int = 64) -> torch.Tensor:
    """Functional form: ``[N,S,M,D] x [L,2] x [N,Lq,M,L,P,2] x [N,Lq,M,L,P] -> [N,Lq,M*D]``."""
    return MSDeformAttnFunction.apply(value, spatial_shapes, sampling_locations, attention_weights, im2col_step)


class MSDeformAttnFusedFunction(Function):
    """The core op with the module's location / softmax arithmetic folded into the kernel prologue (SURVEY 8(f1)):
    ``proj`` is the raw output of the [sampling_offsets | attention_weights] projections, ``reference_points``
    [N, Lq, L, 2]; sampling locations and attention weights are never materialised (ops/modules/ms_deform_attn.py:69-79
    + :86-87 in one launch per direction).  Gradients for ``value`` and ``proj``."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, proj, reference_points, n_points):
        msda = ext.load()
        ctx.n_points = int(n_points)
        out = msda.ms_deform_attn_forward_fused(value, value_spatial_shapes, proj, reference_points, ctx.n_points)
        ctx.save_for_backward(value, value_spatial_shapes, proj, reference_points)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, shapes, proj, ref = ctx.saved_tensors
        gv, gp = ext.load().ms_deform_attn_backward_fused(value, shapes, proj, ref, grad_output.contiguous(), ctx.n_points)
        return gv, None, gp, None, None
