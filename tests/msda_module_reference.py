"""Test helpers for the module-level MSDeformAttn tests: an fp64 restatement of the reference's ``MSDeformAttn.forward``,
kink control for its gradients, and a context that forces one of the module's routes and records the bindings it ran.

* ``msda_fp64`` -- ops/modules/ms_deform_attn.py:60-89 in float64: value projection and padding fill, offsets and
  softmax logits, the ``query_attn_mask`` fill, sampling locations for 2-d references (offsets divided by the level
  sizes as stored, (H, W), like the reference) and 4-d references, the core by ``oracle.torch_ref.msda_core_torch``
  (evaluated in query chunks, recomputed chunk by chunk in the backward so that the fp64 graph of a C2 batch stays
  small), and the output projection.  Gradients come from fp64 autograd.
* ``kinked`` -- bilinear sampling is continuous in the location but its location derivative jumps where a sample's
  pixel coordinate (``x * W - 0.5`` or ``y * H - 0.5``) crosses an integer.  A sample within fp32 rounding of such a
  line can take the one-sided derivative of the neighbouring cell in the kernel and of its own cell in the reference.
  ``kinked`` marks every (image, query) that owns a sample within a few fp32 roundings of one; tests zero the
  upstream gradient there on both sides, so every gradient can be compared tightly and nothing needs a loose group.
* ``forced_route`` -- sets the module's route switches (``TFB200_FUSED_PREP``, ``TFB200_TILED_ENC``,
  ``TFB200_TILED_ENC_BWD``, ``TFB200_TILED_ENC_FUSED``), clears the per-geometry timing caches, and wraps the extension
  so that every ``ms_deform_attn_*`` / ``sampling_prep_*`` binding called is recorded (``BindingSpy``).
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from oracle.torch_ref import msda_core_torch

# Kink margin in pixels on a level side of `side` px: KINK_FLOOR_PX + KINK_PER_PX * side (1e-4 px at 240).  The fp32
# rounding of a sample's pixel coordinate is ~1.2e-7 * side (the location's ulp times the side, plus the rounding of
# x * W - 0.5) plus < 1e-5 px from the offset projection, so the margin is ~3x.  Scaling with the side keeps the share of
# excluded rows near 5 % on eight-level calls (512 coordinates per row) as on four-level ones.
KINK_FLOOR_PX, KINK_PER_PX = 2.5e-5, 3e-7


class _ChunkedCore(torch.autograd.Function):
    """``msda_core_torch`` over query chunks; the backward recomputes each chunk, so only one chunk's grid_sample
    intermediates are alive at a time."""

    @staticmethod
    def forward(ctx, value, loc, attn, hw, chunk):
        ctx.save_for_backward(value, loc, attn)
        ctx.hw, ctx.chunk = hw, chunk
        lq = loc.shape[1]
        return torch.cat([msda_core_torch(value, hw, loc[:, i:i + chunk], attn[:, i:i + chunk])
                          for i in range(0, lq, chunk)], 1)

    @staticmethod
    def backward(ctx, gout):
        value, loc, attn = ctx.saved_tensors
        hw, chunk = ctx.hw, ctx.chunk
        gv, gl, ga = torch.zeros_like(value), torch.empty_like(loc), torch.empty_like(attn)
        for i in range(0, loc.shape[1], chunk):
            with torch.enable_grad():
                v = value.detach().requires_grad_(True)
                lc = loc[:, i:i + chunk].detach().requires_grad_(True)
                at = attn[:, i:i + chunk].detach().requires_grad_(True)
                dv, dl, da = torch.autograd.grad(msda_core_torch(v, hw, lc, at), (v, lc, at), gout[:, i:i + chunk])
            gv += dv
            gl[:, i:i + chunk] = dl
            ga[:, i:i + chunk] = da
        return gv, gl, ga, None, None


def params64(module):
    """The module's parameters as fp64 leaves that collect gradients, keyed by parameter name."""
    return {k: v.detach().double().requires_grad_(True) for k, v in module.named_parameters()}


def _lin(P, name, x):
    return x @ P[name + ".weight"].t() + P[name + ".bias"]


def sampling_locations64(P, query, reference_points, hw, n_heads=8, n_levels=4, n_points=4):
    """fp64 sampling locations [N, Lq, M, L, P, 2] of the module's parameters ``P`` (ms_deform_attn.py:69,76-82)."""
    n, lq, _ = query.shape
    off = _lin(P, "sampling_offsets", query).view(n, lq, n_heads, n_levels, n_points, 2)
    if reference_points.shape[-1] == 2:
        shapes = torch.tensor(hw, dtype=torch.float64, device=query.device)       # (H, W) as stored, like the reference
        return reference_points[:, :, None, :, None, :] + off / shapes[None, None, None, :, None, :]
    return (reference_points[:, :, None, :, None, :2]
            + off / n_points * reference_points[:, :, None, :, None, 2:] * 0.5)


def msda_fp64(P, query, reference_points, input_flatten, hw, input_padding_mask=None, query_attn_mask=None,
              n_heads=8, n_levels=4, n_points=4, chunk=4096):
    """MSDeformAttn.forward of the reference (ops/modules/ms_deform_attn.py:60-89) in fp64.  ``P`` maps parameter names
    to fp64 tensors, ``hw`` is the list of level sizes (H, W); the other arguments are fp64 versions of the module's."""
    n, lq, c = query.shape
    s = input_flatten.shape[1]
    assert sum(h * w for h, w in hw) == s
    value = _lin(P, "value_proj", input_flatten)
    if input_padding_mask is not None:
        value = value.masked_fill(input_padding_mask[..., None], 0.0)
    value = value.view(n, s, n_heads, c // n_heads)
    attn = F.softmax(_lin(P, "attention_weights", query).view(n, lq, n_heads, n_levels * n_points), -1)
    attn = attn.view(n, lq, n_heads, n_levels, n_points)
    if query_attn_mask is not None:
        attn = attn.masked_fill(query_attn_mask[..., None, None, None], 0.0)
    loc = sampling_locations64(P, query, reference_points, hw, n_heads, n_levels, n_points)
    out = _ChunkedCore.apply(value, loc, attn, [tuple(map(int, p)) for p in hw], chunk)
    return _lin(P, "output_proj", out)


def kinked(loc, hw):
    """[N, Lq] mask of the queries owning a sample whose pixel coordinate lies within the kink margin of an integer, i.e.
    of a cell boundary of the bilinear interpolation.  ``loc`` [N, Lq, M, L, P, 2] in fp64."""
    size = torch.tensor([[w, h] for h, w in hw], dtype=torch.float64, device=loc.device)     # (W, H) per level
    delta = KINK_FLOOR_PX + KINK_PER_PX * size[:, None, :]
    px = loc.detach() * size[:, None, :] - 0.5                                              # [N, Lq, M, L, P, 2]
    return ((px - px.round()).abs() < delta).flatten(2).any(-1)


class BindingSpy:
    """Wraps the extension module: forwards every attribute, and records the name and arguments of each
    ``ms_deform_attn_*`` / ``sampling_prep_*`` binding called through it."""

    _RECORDED = ("ms_deform_attn", "sampling_prep")

    def __init__(self, mod):
        self._mod = mod
        self.calls = []

    def __getattr__(self, name):
        fn = getattr(self._mod, name)
        if not (callable(fn) and name.startswith(self._RECORDED)):
            return fn

        def recorded(*args):
            self.calls.append((name, args))
            return fn(*args)
        return recorded

    @property
    def names(self):
        return {name for name, _ in self.calls}

    def prove_tiles(self):
        """Re-run every recorded ``*_enc`` call through its ``*_strict`` binding, which raises instead of falling back
        to the general kernel: the tile kernels did serve those calls."""
        for name, args in self.calls:
            if name in ("ms_deform_attn_forward_enc", "ms_deform_attn_backward_enc"):
                getattr(self._mod, name + "_strict")(*args)
        torch.cuda.synchronize()

    def tiles_refused(self):
        """Names of the recorded ``*_enc`` calls whose geometry the tile kernels reject (the extension fell back)."""
        refused = set()
        for name, args in self.calls:
            if name in ("ms_deform_attn_forward_enc", "ms_deform_attn_backward_enc"):
                try:
                    getattr(self._mod, name + "_strict")(*args)
                except RuntimeError:
                    refused.add(name)
        return refused


@contextlib.contextmanager
def forced_route(fused_prep=False, tiled_enc="0", tiled_enc_bwd="0", tiled_enc_fused="0"):
    """Force the module's routes (the four switches; ``"auto"`` keeps the timed choice) and yield a ``BindingSpy`` that
    records the bindings called.  The timing caches are cleared on entry and on exit, and the switches restored."""
    from trackformer_b200 import ext
    from trackformer_b200 import msda_function as mf
    from trackformer_b200 import msda_module as mm

    def clear():
        mf._ENC_CHOICE.clear()
        mf._ENC_BWD_CHOICE.clear()
        mf._ENC_FUSED_CHOICE.clear()

    saved = (mm._FUSED_PREP, mf._TILED_ENC, mf._TILED_ENC_BWD, mf._TILED_ENC_FUSED, ext.load)
    spy = BindingSpy(ext.load())
    mm._FUSED_PREP, mf._TILED_ENC, mf._TILED_ENC_BWD, mf._TILED_ENC_FUSED = (fused_prep, tiled_enc, tiled_enc_bwd,
                                                                            tiled_enc_fused)
    ext.load = lambda: spy
    clear()
    try:
        yield spy
    finally:
        mm._FUSED_PREP, mf._TILED_ENC, mf._TILED_ENC_BWD, mf._TILED_ENC_FUSED, ext.load = saved
        clear()
