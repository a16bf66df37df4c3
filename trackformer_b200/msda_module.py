"""``MSDeformAttn`` -- the multi-scale deformable attention layer on the H100 kernels.

Mirror of the reference module (src/trackformer/models/ops/modules/ms_deform_attn.py:15-89):
same constructor, same sub-module names (``sampling_offsets``, ``attention_weights``, ``value_proj``,
``output_proj`` -- checkpoints and the name-based optimiser groups of src/train.py:101-110 keep
working), same ``forward`` signature and the same arithmetic, including the reference's
normalisation of the (x, y) offsets by ``input_spatial_shapes`` as stored, i.e. (H, W)
(ms_deform_attn.py:78-79).

Host-side differences (results identical up to fp32 rounding):
  * the two query projections (offsets: 2*M*L*P outputs, weights: M*L*P outputs) run as ONE GEMM over
    the concatenated weight -- one pass over ``query`` instead of two;
  * the core op is :class:`trackformer_b200.msda_function.MSDeformAttnFunction` (CUDA only, no fallback).
"""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F
from torch import nn

from .fused_linear import linear as fused_linear
from .msda_function import (MSDeformAttnEncFunction, MSDeformAttnEncFusedFunction, MSDeformAttnFunction,
                            MSDeformAttnFusedFunction, encoder_fused_choice)

# fold sampling_prep into the MSDeformAttn kernels (csrc/msda_run.cuh PREP variants)
_FUSED_PREP = os.environ.get("TFB200_FUSED_PREP", "0") != "0"

# the 8 compass directions the reference seeds the per-head offset bias with (ms_deform_attn.py:36)
_COMPASS = ((-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1))


class _SamplingPrep(torch.autograd.Function):
    """[offsets | logits] projection -> (sampling locations, softmax attention weights) in one fused kernel
    (csrc/fused_norm.cu).  Used when the reference points carry no gradient (encoder; decoder layers after the first)."""

    @staticmethod
    def forward(ctx, proj, ref, shapes_f32, m, lv, pt):
        from . import ext
        loc, attn = ext.load().sampling_prep_forward(proj, ref, shapes_f32, m, lv, pt)
        ctx.save_for_backward(attn, ref, shapes_f32)
        ctx.dims = (m, lv, pt)
        return loc, attn

    @staticmethod
    def backward(ctx, grad_loc, grad_attn):
        from . import ext
        attn, ref, shapes_f32 = ctx.saved_tensors
        m, lv, pt = ctx.dims
        gp = ext.load().sampling_prep_backward(grad_loc, grad_attn, attn, ref, shapes_f32, m, lv, pt)
        return gp, None, None, None, None, None


class MSDeformAttn(nn.Module):
    def __init__(self, d_model: int = 256, n_levels: int = 4, n_heads: int = 8, n_points: int = 4,
                 im2col_step: int = 64):
        super().__init__()
        if d_model % n_heads != 0:
            raise AssertionError("d_model must be divisible by n_heads")
        self.im2col_step = im2col_step
        self.d_model = d_model
        self.n_levels = n_levels
        self.n_heads = n_heads
        self.n_points = n_points

        self.sampling_offsets = nn.Linear(d_model, n_heads * n_levels * n_points * 2)
        self.attention_weights = nn.Linear(d_model, n_heads * n_levels * n_points)
        self.value_proj = nn.Linear(d_model, d_model)
        self.output_proj = nn.Linear(d_model, d_model)
        self._reset_parameters()

    def _reset_parameters(self):
        """Reference init (ms_deform_attn.py:33-47): zero offset weights, compass-grid offset bias scaled
        by the point index, zero attention logits, xavier value/output projections."""
        with torch.no_grad():
            for lin in (self.sampling_offsets, self.attention_weights):
                lin.weight.zero_()
            self.attention_weights.bias.zero_()
            # head h looks along compass direction h; its k-th point sits k+1 steps out, on every level
            steps = torch.arange(1, self.n_points + 1, dtype=torch.float32).view(1, 1, self.n_points, 1)
            rays = torch.tensor(_COMPASS, dtype=torch.float32).view(self.n_heads, 1, 1, 2)   # the reference hard-codes 8 heads
            self.sampling_offsets.bias = nn.Parameter((rays * steps).expand(-1, self.n_levels, -1, -1).reshape(-1))
            for lin in (self.value_proj, self.output_proj):
                nn.init.xavier_uniform_(lin.weight)
                lin.bias.zero_()

    @staticmethod
    def _float_shapes(spatial_shapes, like):
        """``spatial_shapes`` as floats, memoised on the (cached) shapes tensor.  Dividing by it gives the same quotient as
        dividing by the int64 tensor (type promotion converts that to float32 first) but keeps TensorIterator on its
        vectorised same-dtype path (35 -> ~8 us per C2 encoder call)."""
        f = getattr(spatial_shapes, "_as_float", None)
        if f is None or f.dtype != like.dtype:
            f = spatial_shapes.to(like.dtype)
            try:
                spatial_shapes._as_float = f
            except AttributeError:
                pass
        return f

    def _sampling_locations(self, reference_points, offsets, spatial_shapes):
        """Normalised (x, y) of every sample: reference point + offset.  2-d references: offsets are in pixels of the
        level, divided by ``spatial_shapes`` as stored -- (H, W), like the reference (ms_deform_attn.py:78-79);
        4-d references (boxes): offsets are fractions of half the box size, split over the points (:80-82)."""
        kind = reference_points.shape[-1]
        if kind == 2:
            divisor = self._float_shapes(spatial_shapes, offsets)
            return reference_points[:, :, None, :, None, :] + offsets / divisor[None, None, None, :, None, :]
        if kind == 4:
            centre, size = reference_points[:, :, None, :, None, :2], reference_points[:, :, None, :, None, 2:]
            return centre + offsets / self.n_points * size * 0.5
        raise ValueError("Last dim of reference_points must be 2 or 4, but get {} instead.".format(kind))

    def forward(self, query, reference_points, input_flatten, input_spatial_shapes,
                input_padding_mask=None, query_attn_mask=None):
        """query [N,Lq,C]; reference_points [N,Lq,L,2|4] in [0,1] over the padded extent;
        input_flatten [N,S,C]; input_spatial_shapes [L,2]=(H,W) int64; input_padding_mask [N,S] True=pad.
        Returns [N,Lq,C]."""
        n, len_q, _ = query.shape
        len_in = input_flatten.shape[1]
        heads, levels, points = self.n_heads, self.n_levels, self.n_points
        hw = getattr(input_spatial_shapes, "_hw_list", None)      # host copy attached by the transformer
        if hw is not None:
            assert sum(h * w for h, w in hw) == len_in
        else:                                                       # reference behaviour: device reduction + sync
            assert int((input_spatial_shapes[:, 0] * input_spatial_shapes[:, 1]).sum()) == len_in

        value = fused_linear(input_flatten, self.value_proj.weight, self.value_proj.bias)
        if input_padding_mask is not None:
            value = value.masked_fill(input_padding_mask[..., None], 0.0)
        value = value.view(n, len_in, heads, self.d_model // heads)

        # one GEMM for [offsets | logits]
        n_off = heads * levels * points * 2
        proj = fused_linear(query, torch.cat([self.sampling_offsets.weight, self.attention_weights.weight], 0),
                            torch.cat([self.sampling_offsets.bias, self.attention_weights.bias], 0))
        lp = levels * points
        d_head = self.d_model // heads
        if (_FUSED_PREP and proj.is_cuda and proj.dtype == torch.float32 and query_attn_mask is None
                and not reference_points.requires_grad and reference_points.shape[-1] == 2 and lp == 16
                and d_head in (32, 36) and heads % 4 == 0 and n * len_q * heads > 32768 and len_q >= 2048):
            # encoder-sized call: softmax + location arithmetic inside the gather kernel's prologue, sampling locations
            # and attention weights never touch HBM (ms_deform_attn.py:69-87 as one launch per direction)
            out = MSDeformAttnFusedFunction.apply(value, input_spatial_shapes, proj, reference_points, points)
            return fused_linear(out, self.output_proj.weight, self.output_proj.bias)
        if (hw is not None and len_q == len_in and proj.is_cuda and proj.dtype == torch.float32 and query_attn_mask is None
                and not reference_points.requires_grad and reference_points.shape[-1] == 2 and levels == 4 and points == 4
                and d_head == 32):
            # encoder call: the TMA tile kernels can evaluate softmax + locations in their tap pass; taken when that beats
            # "sampling-prep kernel + op" on this geometry (timed once on the first eager call)
            flat_hw = [int(v) for pair in hw for v in pair]
            key = (tuple(value.shape), tuple(flat_hw), value.device.index)

            def unfused():
                with torch.no_grad():
                    lc, at = _SamplingPrep.apply(proj, reference_points, self._float_shapes(input_spatial_shapes, proj),
                                                 heads, levels, points)
                    return MSDeformAttnEncFunction.apply(value, input_spatial_shapes, lc, at, self.im2col_step)

            def fused():
                with torch.no_grad():
                    return MSDeformAttnEncFusedFunction.apply(value, proj, reference_points, flat_hw)
            if encoder_fused_choice(key, fused, unfused):
                out = MSDeformAttnEncFusedFunction.apply(value, proj, reference_points, flat_hw)
                return fused_linear(out, self.output_proj.weight, self.output_proj.bias)
        fusable = (proj.is_cuda and proj.dtype == torch.float32 and query_attn_mask is None
                   and not reference_points.requires_grad and reference_points.shape[-1] in (2, 4)
                   and lp in (4, 8, 16, 32) and (heads * lp) % 32 == 0)
        if fusable:
            # softmax + offset normalisation + reference add in one pass over proj (ms_deform_attn.py:69-82)
            locations, attn = _SamplingPrep.apply(proj, reference_points, self._float_shapes(input_spatial_shapes, proj),
                                                  heads, levels, points)
        else:
            offsets = proj[..., :n_off].reshape(n, len_q, heads, levels, points, 2)
            attn = F.softmax(proj[..., n_off:].reshape(n, len_q, heads, lp), -1).view(n, len_q, heads, levels, points)
            if query_attn_mask is not None:
                attn = attn.masked_fill(query_attn_mask[..., None, None, None], 0.0)
            locations = self._sampling_locations(reference_points, offsets, input_spatial_shapes)

        if hw is not None and len_q == len_in and value.is_cuda and value.dtype == torch.float32:
            # encoder self-attention: queries are the pixels -> the TMA-staged tile kernel is a candidate (chosen per
            # geometry by a one-time measurement, msda_function.encoder_kernel_choice)
            core = MSDeformAttnEncFunction
        else:
            core = MSDeformAttnFunction
        out = core.apply(value, input_spatial_shapes, locations, attn, self.im2col_step)
        return fused_linear(out, self.output_proj.weight, self.output_proj.bias)
