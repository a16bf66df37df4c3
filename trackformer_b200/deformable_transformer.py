"""Deformable transformer (6 encoder + 6 decoder layers) on the H100 MSDeformAttn kernels.

Mirror of src/trackformer/models/deformable_transformer.py (one-stage path, which is what every shipped
config uses -- cfgs/train_deformable.yaml sets ``with_box_refine: true`` and leaves ``two_stage: false``):

  DeformableTransformer.forward(srcs, masks, pos_embeds, query_embed, targets)       :133-255
  encoder layer / encoder (+ reference-point grid)                                    :258-327
  decoder layer / decoder (+ iterative box refinement, detached)                      :330-431
  track-query concatenation [prev hs_embed ; query tgt], zero query_pos for tracks    :202-225
  separate prev/current-frame encoder passes for multi-frame attention                :160-173

  two-stage: encoder proposals, encoder head, top-k query selection and sine query embedding    :77-122,180-194

Module and parameter names equal the reference's, so ``state_dict`` round-trips.  Two-stage runs on CUDA through
csrc/two_stage.cu (one launch for the proposals and the masked memory, one for the selection, its embedding and the
reference points) and on the CPU as the reference's torch ops; it does not take track queries or separate per-frame
encoders (the detector classes refuse those combinations).
"""
from __future__ import annotations

import copy
import math
import os

import torch
import torch.nn.functional as F
from torch import nn

from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import seeds, small_attention
from .fused_linear import ffn, ffn_fusable, linear as fused_linear, relu_dropout
from .fused_norm import add_dropout_layernorm
from .msda_module import MSDeformAttn
from .util import refine_boxes


def _clones(module: nn.Module, n: int) -> nn.ModuleList:
    return nn.ModuleList([copy.deepcopy(module) for _ in range(n)])


def _activation(name: str):
    try:
        return {"relu": F.relu, "gelu": F.gelu, "glu": F.glu}[name]
    except KeyError:
        raise RuntimeError(f"activation should be relu/gelu, not {name}.") from None


def _add_pos(x, pos):
    return x if pos is None else x + pos


# A/B switch (measurement only): True forces nn.MultiheadAttention's unfused bmm / softmax / bmm path
_MHA_NEED_WEIGHTS = os.environ.get("TFB200_MHA_NEED_WEIGHTS", "0") == "1"


def proposal_dim_t(device) -> torch.Tensor:
    """The 128 frequencies of get_proposal_pos_embed (:93-95), computed by torch as the reference computes them."""
    dim_t = torch.arange(128, dtype=torch.float32)
    return (10000 ** (2 * (dim_t // 2) / 128)).to(device)


def proposal_pos_embed(proposals: torch.Tensor) -> torch.Tensor:
    """[N, L, 4] unactivated boxes -> [N, L, 512] sine embedding (deformable_transformer.py:89-102)."""
    dim_t = proposal_dim_t(proposals.device)
    proposals = proposals.sigmoid() * (2 * math.pi)
    pos = proposals[:, :, :, None] / dim_t
    return torch.stack((pos[:, :, :, 0::2].sin(), pos[:, :, :, 1::2].cos()), dim=4).flatten(2)


def encoder_output_proposals(memory, padding_mask, hw):
    """(masked memory, proposal logits [N, S, 4]) of gen_encoder_output_proposals (:104-133) without its encoder head;
    ``padding_mask`` [N, S] (True = padded) or None for an unpadded batch.  The torch route (CPU, non-fp32)."""
    n = memory.shape[0]
    if padding_mask is None:
        padding_mask = torch.zeros(memory.shape[:2], dtype=torch.bool, device=memory.device)
    proposals, cur = [], 0
    for lvl, (h, w) in enumerate(hw):
        m = padding_mask[:, cur:cur + h * w].view(n, h, w, 1)
        valid_h = torch.sum(~m[:, :, 0, 0], 1)
        valid_w = torch.sum(~m[:, 0, :, 0], 1)
        gy, gx = torch.meshgrid(torch.linspace(0, h - 1, h, dtype=torch.float32, device=memory.device),
                                torch.linspace(0, w - 1, w, dtype=torch.float32, device=memory.device), indexing="ij")
        grid = torch.cat([gx.unsqueeze(-1), gy.unsqueeze(-1)], -1)
        scale = torch.cat([valid_w.unsqueeze(-1), valid_h.unsqueeze(-1)], 1).view(n, 1, 1, 2)
        grid = (grid.unsqueeze(0).expand(n, -1, -1, -1) + 0.5) / scale
        wh = torch.ones_like(grid) * 0.05 * (2.0 ** lvl)
        proposals.append(torch.cat((grid, wh), -1).view(n, -1, 4))
        cur += h * w
    out = torch.cat(proposals, 1)
    valid = ((out > 0.01) & (out < 0.99)).all(-1, keepdim=True)
    out = torch.log(out / (1 - out))
    out = out.masked_fill(padding_mask.unsqueeze(-1), float("inf")).masked_fill(~valid, float("inf"))
    masked = memory.masked_fill(padding_mask.unsqueeze(-1), 0.0).masked_fill(~valid, 0.0)
    return masked, out


class _MaskedMemory(Function):
    """memory -> (memory with the invalid proposal rows zeroed, proposal logits, valid flags) on CUDA: one launch of the
    proposal kernel, or -- with ``memo`` = (proposal logits, flags) of an unpadded geometry -- of the row mask alone.
    The gradient is masked the same way (one launch)."""

    @staticmethod
    def forward(ctx, memory, padding_mask, hw_flat, memo):
        from . import ext
        m = ext.load()
        if memo is not None:
            prop, valid = memo
            masked = m.two_stage_mask_rows(memory, valid)
        else:
            prop, valid, masked = m.two_stage_proposals(padding_mask, memory, hw_flat, memory.shape[0],
                                                        memory.device.index)
        ctx.save_for_backward(valid)
        ctx.mark_non_differentiable(prop, valid)
        return masked, prop, valid

    @staticmethod
    @once_differentiable
    def backward(ctx, g_masked, _g_prop, _g_valid):
        from . import ext
        valid, = ctx.saved_tensors
        return ext.load().two_stage_mask_rows(g_masked.contiguous(), valid), None, None, None


class DeformableTransformerEncoderLayer(nn.Module):
    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8,
                 n_points=4):
        super().__init__()
        self.self_attn = MSDeformAttn(d_model, n_levels, n_heads, n_points)
        self.dropout1 = nn.Dropout(dropout)
        self.norm1 = nn.LayerNorm(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.activation = _activation(activation)
        self.dropout2 = nn.Dropout(dropout)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.dropout3 = nn.Dropout(dropout)
        self.norm2 = nn.LayerNorm(d_model)

    with_pos_embed = staticmethod(_add_pos)

    def forward_ffn(self, src):
        if self.activation is F.relu and ffn_fusable(src, self.linear1, self.linear2, self.dropout2):
            ff = ffn(src, self.linear1, self.linear2, self.dropout2)
        else:
            a = fused_linear(src, self.linear1.weight, self.linear1.bias)
            h = relu_dropout(a, self.dropout2) if self.activation is F.relu else self.dropout2(self.activation(a))
            ff = fused_linear(h, self.linear2.weight, self.linear2.bias)
        return add_dropout_layernorm(src, ff, self.dropout3, self.norm2)

    def forward(self, src, pos, reference_points, spatial_shapes, padding_mask=None):
        attn = self.self_attn(_add_pos(src, pos), reference_points, src, spatial_shapes, padding_mask)
        src = add_dropout_layernorm(src, attn, self.dropout1, self.norm1)
        return self.forward_ffn(src)


class DeformableTransformerEncoder(nn.Module):
    def __init__(self, encoder_layer, num_layers):
        super().__init__()
        self.layers = _clones(encoder_layer, num_layers)
        self.num_layers = num_layers
        self._ref_memo = {}

    @staticmethod
    def get_reference_points(spatial_shapes, valid_ratios, device):
        """Pixel centres of every level, normalised by the valid extent, then expressed in every level's
        frame: [N, S, L, 2] (deformable_transformer.py:306-319)."""
        hw = getattr(spatial_shapes, "_hw_list", None) or [(int(h), int(w)) for h, w in spatial_shapes.tolist()]
        per_level = []
        for lvl, (h, w) in enumerate(hw):
            ys = torch.linspace(0.5, h - 0.5, h, dtype=torch.float32, device=device)
            xs = torch.linspace(0.5, w - 0.5, w, dtype=torch.float32, device=device)
            gy, gx = torch.meshgrid(ys, xs, indexing="ij")
            ry = gy.reshape(-1)[None] / (valid_ratios[:, None, lvl, 1] * h)
            rx = gx.reshape(-1)[None] / (valid_ratios[:, None, lvl, 0] * w)
            per_level.append(torch.stack((rx, ry), -1))
        ref = torch.cat(per_level, 1)
        return ref[:, :, None] * valid_ratios[:, None]

    def forward(self, src, spatial_shapes, valid_ratios, pos=None, padding_mask=None):
        hw = getattr(spatial_shapes, "_hw_list", None)
        if hw is not None and padding_mask is None:
            # dense batch (valid ratios are exactly 1): the grid depends on the level sizes only -- memoise it
            key = (tuple(hw), src.shape[0], src.device)
            ref = self._ref_memo.get(key)
            if ref is None:
                ref = self._ref_memo[key] = self.get_reference_points(spatial_shapes, valid_ratios, src.device)
        else:
            ref = self.get_reference_points(spatial_shapes, valid_ratios, device=src.device)
        out = src
        for layer in self.layers:
            out = layer(out, pos, ref, spatial_shapes, padding_mask)
        return out


class DeformableTransformerDecoderLayer(nn.Module):
    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8,
                 n_points=4):
        super().__init__()
        self.cross_attn = MSDeformAttn(d_model, n_levels, n_heads, n_points)
        self.dropout1 = nn.Dropout(dropout)
        self.norm1 = nn.LayerNorm(d_model)
        self.self_attn = nn.MultiheadAttention(d_model, n_heads, dropout=dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.norm2 = nn.LayerNorm(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.activation = _activation(activation)
        self.dropout3 = nn.Dropout(dropout)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.dropout4 = nn.Dropout(dropout)
        self.norm3 = nn.LayerNorm(d_model)

    with_pos_embed = staticmethod(_add_pos)

    def forward_ffn(self, tgt):
        # fused_linear: F.linear whose bias gradient is one column-sum launch (the generic reduction: 7-16 us per call)
        h = self.dropout3(self.activation(fused_linear(tgt, self.linear1.weight, self.linear1.bias)))
        ff = fused_linear(h, self.linear2.weight, self.linear2.bias)
        return add_dropout_layernorm(tgt, ff, self.dropout4, self.norm3)

    def forward(self, tgt, query_pos, reference_points, src, src_spatial_shapes, src_padding_mask=None,
                query_attn_mask=None, padded_queries=None):
        # query self-attention (dense, tiny: Lq <= ~800) -- sequence-first nn.MultiheadAttention like the reference.
        # padded_queries [N, Lq] marks filler queries (fixed-shape CUDA-graph replays, graphed_detector.py): they are
        # hidden from the real queries as attention KEYS, which is all it takes for the real rows to be unaffected
        # (every other decoder op is row-wise).
        qk = _add_pos(tgt, query_pos).transpose(0, 1)
        key_mask = query_attn_mask if padded_queries is None else padded_queries
        # need_weights=False: the averaged attention map is never used (the reference discards it too,
        # deformable_transformer.py:368) and asking for it forces the unfused bmm / softmax / bmm path with ~25 small
        # launches per layer and direction; without it the module runs one fused attention kernel
        if small_attention.supported(self.self_attn, qk) and not _MHA_NEED_WEIGHTS:
            sa = small_attention.mha_forward(self.self_attn, qk, tgt.transpose(0, 1), key_mask).transpose(0, 1)
        else:
            sa = self.self_attn(qk, qk, tgt.transpose(0, 1), key_padding_mask=key_mask,
                                need_weights=_MHA_NEED_WEIGHTS)[0].transpose(0, 1)
        tgt = add_dropout_layernorm(tgt, sa, self.dropout2, self.norm2)
        # deformable cross-attention into the encoder memory
        ca = self.cross_attn(_add_pos(tgt, query_pos), reference_points, src, src_spatial_shapes,
                             src_padding_mask, query_attn_mask)
        tgt = add_dropout_layernorm(tgt, ca, self.dropout1, self.norm1)
        return self.forward_ffn(tgt)


class DeformableTransformerDecoder(nn.Module):
    def __init__(self, decoder_layer, num_layers, return_intermediate=False):
        super().__init__()
        self.layers = _clones(decoder_layer, num_layers)
        self.num_layers = num_layers
        self.return_intermediate = return_intermediate
        self.bbox_embed = None     # set by DeformableDETR for iterative box refinement
        self.class_embed = None

    def forward(self, tgt, reference_points, src, src_spatial_shapes, src_valid_ratios, query_pos=None,
                src_padding_mask=None, query_attn_mask=None, padded_queries=None):
        out = tgt
        hs, refs, boxes = [], [], []
        self.refined_boxes = None
        for lid, layer in enumerate(self.layers):
            if reference_points.shape[-1] == 4:
                ref_in = reference_points[:, :, None] * torch.cat([src_valid_ratios, src_valid_ratios], -1)[:, None]
            else:
                assert reference_points.shape[-1] == 2
                ref_in = reference_points[:, :, None] * src_valid_ratios[:, None]
            out = layer(out, query_pos, ref_in, src, src_spatial_shapes, src_padding_mask, query_attn_mask,
                        padded_queries)

            if self.bbox_embed is not None:     # refine the reference boxes for the next layer; no gradient through them
                # sigmoid(bbox_embed[lid](out) + inverse_sigmoid(reference)) is ALSO what the detection head of this
                # layer predicts (deformable_detr.py:229-248 evaluates the same MLP on the same input a second time):
                # keep the attached tensor for the heads, continue with its detached value
                refined = refine_boxes(self.bbox_embed[lid](out), reference_points)
                boxes.append(refined)
                reference_points = refined.detach()

            if self.return_intermediate:
                hs.append(out)
                refs.append(reference_points)
        if self.return_intermediate:
            if boxes:
                self.refined_boxes = torch.stack(boxes)      # [layers, N, Q, 4], attached; consumed once by the heads
            return torch.stack(hs), torch.stack(refs)
        return out, reference_points


class DeformableTransformer(nn.Module):
    def __init__(self, d_model=256, nhead=8, num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=1024,
                 dropout=0.1, activation="relu", return_intermediate_dec=False, num_feature_levels=4,
                 dec_n_points=4, enc_n_points=4, two_stage=False, two_stage_num_proposals=300,
                 multi_frame_attention_separate_encoder=False):
        super().__init__()
        if two_stage and multi_frame_attention_separate_encoder:
            raise NotImplementedError("two-stage Deformable DETR with multi-frame attention: the proposal widths would "
                                      "grow over both frames' levels")
        self.d_model = d_model
        self.nhead = nhead
        self.two_stage = two_stage
        self.two_stage_num_proposals = two_stage_num_proposals
        self.num_feature_levels = num_feature_levels
        self.multi_frame_attention_separate_encoder = multi_frame_attention_separate_encoder

        enc_levels = num_feature_levels // 2 if multi_frame_attention_separate_encoder else num_feature_levels
        self.encoder = DeformableTransformerEncoder(
            DeformableTransformerEncoderLayer(d_model, dim_feedforward, dropout, activation, enc_levels, nhead,
                                              enc_n_points), num_encoder_layers)
        self.decoder = DeformableTransformerDecoder(
            DeformableTransformerDecoderLayer(d_model, dim_feedforward, dropout, activation, num_feature_levels,
                                              nhead, dec_n_points), num_decoder_layers, return_intermediate_dec)
        self.level_embed = nn.Parameter(torch.Tensor(num_feature_levels, d_model))
        if two_stage:
            self.enc_output = nn.Linear(d_model, d_model)
            self.enc_output_norm = nn.LayerNorm(d_model)
            self.pos_trans = nn.Linear(d_model * 2, d_model * 2)
            self.pos_trans_norm = nn.LayerNorm(d_model * 2)
        else:
            self.reference_points = nn.Linear(d_model, 2)
        self.selected_tokens = None         # two-stage: [N, k] token indices chosen by the latest forward
        self._shapes_memo = {}
        self._proposal_memo = {}
        self._reset_parameters()

    def _reset_parameters(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for mod in self.modules():
            if isinstance(mod, MSDeformAttn):
                mod._reset_parameters()
        if not self.two_stage:
            nn.init.xavier_uniform_(self.reference_points.weight, gain=1.0)
            nn.init.zeros_(self.reference_points.bias)
        nn.init.normal_(self.level_embed)

    def _shapes_tensor(self, hw, device):
        """[L,2] int64 (H,W) on the device, built once per geometry (no per-forward H2D copy, graph-capture safe);
        the host copy rides along as ``_hw_list`` so that callees never have to sync to learn the level sizes."""
        key = (tuple(hw), device)
        t = self._shapes_memo.get(key)
        if t is None:
            t = torch.as_tensor(hw, dtype=torch.long, device=device)
            t._hw_list = list(hw)
            self._shapes_memo[key] = t
        return t

    @staticmethod
    def get_valid_ratio(mask):
        """Fraction of each padded level that holds image content, as (w, h)."""
        _, h, w = mask.shape
        if getattr(mask, "_no_padding", False):
            return torch.ones(mask.shape[0], 2, dtype=torch.float32, device=mask.device)
        vh = (~mask[:, :, 0]).sum(1).float() / h
        vw = (~mask[:, 0, :]).sum(1).float() / w
        return torch.stack([vw, vh], -1)

    def _unit_ratios(self, batch, levels, device):
        key = (batch, levels, device)
        memo = self.__dict__.setdefault("_unit_ratio_memo", {})
        hit = memo.get(key)
        if hit is None or torch.is_inference_mode_enabled():
            hit = torch.ones(batch, levels, 2, dtype=torch.float32, device=device)
            if not torch.is_inference_mode_enabled():
                memo[key] = hit
        return hit

    def _proposals(self, memory, enc_mask, hw):
        """(masked memory, proposal logits) of the encoder output: the kernels on CUDA fp32, the reference's ops
        elsewhere.  An unpadded batch's proposals depend on its geometry only and are made once."""
        if not (memory.is_cuda and memory.dtype == torch.float32):
            return encoder_output_proposals(memory, enc_mask, hw)
        hw_flat = [v for pair in hw for v in pair]
        memo = None
        if enc_mask is None:
            key = (tuple(hw), memory.shape[0], memory.device)
            memo = self._proposal_memo.get(key)
            if memo is None or torch.is_inference_mode_enabled():
                from . import ext
                # made on the memory's device, whichever device is current
                prop, valid, _ = ext.load().two_stage_proposals(None, None, hw_flat, memory.shape[0],
                                                                memory.device.index)
                memo = (prop, valid)
                if not torch.is_inference_mode_enabled():
                    self._proposal_memo[key] = memo
        masked, prop, _ = _MaskedMemory.apply(memory.contiguous(), enc_mask, hw_flat, memo)
        return masked, prop

    def _dim_t(self, device):
        memo = self.__dict__.setdefault("_dim_t_memo", {})
        t = memo.get(device)
        if t is None or torch.is_inference_mode_enabled():
            t = proposal_dim_t(device)
            if not torch.is_inference_mode_enabled():
                memo[device] = t
        return t

    def two_stage_queries(self, memory, enc_mask, hw):
        """Encoder head, top-k selection and query embedding of deformable_transformer.py:180-194 ->
        (query_pos, tgt, reference boxes [N, k, 4], encoder class logits [N, S, C], unactivated boxes [N, S, 4])."""
        masked, proposals = self._proposals(memory, enc_mask, hw)
        out_memory = self.enc_output_norm(fused_linear(masked, self.enc_output.weight, self.enc_output.bias))
        last = self.decoder.num_layers
        head = self.decoder.class_embed[last]
        enc_class = fused_linear(out_memory, head.weight, head.bias)
        enc_unact = self.decoder.bbox_embed[last](out_memory) + proposals
        k = self.two_stage_num_proposals
        if enc_class.is_cuda and enc_class.dtype == torch.float32:
            from . import ext
            idx, boxes, reference, embed = ext.load().two_stage_select(enc_class.detach(), enc_unact.detach(),
                                                                      self._dim_t(enc_class.device), k)
        else:
            idx = torch.topk(enc_class[..., 0], k, dim=1)[1]
            boxes = torch.gather(enc_unact, 1, idx.unsqueeze(-1).repeat(1, 1, 4)).detach()
            reference = boxes.sigmoid()
            embed = proposal_pos_embed(boxes)
        self.selected_tokens = idx
        pos_trans_out = self.pos_trans_norm(fused_linear(embed, self.pos_trans.weight, self.pos_trans.bias))
        query_pos, tgt = torch.split(pos_trans_out, memory.shape[-1], dim=2)
        return query_pos, tgt, reference, enc_class, enc_unact

    def forward(self, srcs, masks, pos_embeds, query_embed=None, targets=None):
        """-> (hs, memory, init_reference, inter_references, refined boxes or None, encoder outputs): the last is None,
        or with two-stage (class logits [N, S, C], unactivated boxes [N, S, 4]) of the encoder head."""
        assert self.two_stage or query_embed is not None
        if self.training and srcs[0].is_cuda:
            seeds.begin_step(srcs[0].device)      # one launch draws the dropout seeds of every fused site of this pass
        hw, src_l, pos_l = [], [], []
        for lvl, (src, pos) in enumerate(zip(srcs, pos_embeds)):
            hw.append((int(src.shape[2]), int(src.shape[3])))
            src_l.append(src.flatten(2).transpose(1, 2))
            pos_l.append(pos.flatten(2).transpose(1, 2) + self.level_embed[lvl].view(1, 1, -1))
        src_flat = torch.cat(src_l, 1)
        pos_flat = torch.cat(pos_l, 1)
        spatial_shapes = self._shapes_tensor(hw, src_flat.device)
        dense = all(getattr(m, "_no_padding", False) for m in masks)
        if dense:                                        # no padding anywhere: unit valid ratios, and an all-False
            enc_mask = None                              # mask is a no-op in MSDeformAttn -> nothing to build
            valid_ratios = self._unit_ratios(src_flat.shape[0], len(masks), src_flat.device)
        else:
            enc_mask = torch.cat([m.flatten(1) for m in masks], 1)
            valid_ratios = torch.stack([self.get_valid_ratio(m) for m in masks], 1)
        if self.multi_frame_attention_separate_encoder:
            half_s, half_l = src_flat.shape[1] // 2, self.num_feature_levels // 2

            def _enc(sl_s, sl_l):
                shp = self._shapes_tensor(hw[sl_l], src_flat.device)
                return self.encoder(src_flat[:, sl_s], shp, valid_ratios[:, sl_l], pos_flat[:, sl_s],
                                    None if enc_mask is None else enc_mask[:, sl_s])
            prev_memory = _enc(slice(None, half_s), slice(None, half_l))
            memory = _enc(slice(half_s, None), slice(half_l, None))
            memory = torch.cat([memory, prev_memory], 1)
        else:
            memory = self.encoder(src_flat, spatial_shapes, valid_ratios, pos_flat, enc_mask)

        bs, _, c = memory.shape
        padded_queries = enc_outputs = None
        if self.two_stage:
            query_pos, tgt, reference_points, enc_class, enc_unact = self.two_stage_queries(memory, enc_mask, hw)
            enc_outputs = (enc_class, enc_unact)
        else:
            query_pos, tgt = torch.split(query_embed, c, dim=1)
            query_pos = query_pos.unsqueeze(0).expand(bs, -1, -1)
            tgt = tgt.unsqueeze(0).expand(bs, -1, -1)
            reference_points = self.reference_points(query_pos).sigmoid()

        if not self.two_stage and targets is not None and "track_query_hs_embeds" in targets[0]:
            # track queries: previous-frame output embeddings as content, zero positional part, previous box
            # centres as reference points; they are prepended to the object queries
            prev_hs = torch.stack([t["track_query_hs_embeds"] for t in targets])
            prev_boxes = torch.stack([t["track_query_boxes"] for t in targets])
            query_pos = torch.cat([torch.zeros_like(prev_hs), query_pos], dim=1)
            tgt = torch.cat([prev_hs, tgt], dim=1)
            reference_points = torch.cat([prev_boxes[..., :2], reference_points], dim=1)
            if "track_query_padding" in targets[0]:
                # [K] bool per image, True = filler track query (not in the reference: used by GraphedDetector)
                filler = torch.stack([t["track_query_padding"] for t in targets])
                padded_queries = torch.cat([filler, filler.new_zeros(bs, tgt.shape[1] - filler.shape[1])], dim=1)
        init_reference = reference_points

        hs, inter_references = self.decoder(tgt, reference_points, memory, spatial_shapes, valid_ratios,
                                            query_pos, enc_mask, None, padded_queries)
        refined, self.decoder.refined_boxes = self.decoder.refined_boxes, None     # (do not keep the graph alive)
        return hs, memory, init_reference, inter_references, refined, enc_outputs


def build_deforamble_transformer(args):
    """(sic) -- the reference spells it this way, models/__init__.py:7."""
    levels = args.num_feature_levels * (2 if args.multi_frame_attention else 1)
    return DeformableTransformer(
        d_model=args.hidden_dim, nhead=args.nheads, num_encoder_layers=args.enc_layers,
        num_decoder_layers=args.dec_layers, dim_feedforward=args.dim_feedforward, dropout=args.dropout,
        activation="relu", return_intermediate_dec=True, num_feature_levels=levels,
        dec_n_points=args.dec_n_points, enc_n_points=args.enc_n_points, two_stage=args.two_stage,
        two_stage_num_proposals=args.num_queries,
        multi_frame_attention_separate_encoder=args.multi_frame_attention and args.multi_frame_attention_separate_encoder)
