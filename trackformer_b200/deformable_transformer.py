"""Deformable transformer (6 encoder + 6 decoder layers) on the H100 MSDeformAttn kernels.

Mirror of src/trackformer/models/deformable_transformer.py (one-stage path, which is what every shipped
config uses -- cfgs/train_deformable.yaml sets ``with_box_refine: true`` and leaves ``two_stage: false``):

  DeformableTransformer.forward(srcs, masks, pos_embeds, query_embed, targets)       :133-255
  encoder layer / encoder (+ reference-point grid)                                    :258-327
  decoder layer / decoder (+ iterative box refinement, detached)                      :330-431
  track-query concatenation [prev hs_embed ; query tgt], zero query_pos for tracks    :202-225
  separate prev/current-frame encoder passes for multi-frame attention                :160-173

Module and parameter names equal the reference's, so ``state_dict`` round-trips.  Two-stage proposal
generation (:77-122,:180-194) is not on the hot path of any shipped configuration and is not built.
"""
from __future__ import annotations

import copy

import os

import torch
import torch.nn.functional as F
from torch import nn

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
        if two_stage:
            raise NotImplementedError("two-stage Deformable-DETR is outside the hot path (no shipped config uses it)")
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
        self.reference_points = nn.Linear(d_model, 2)
        self._shapes_memo = {}
        self._reset_parameters()

    def _reset_parameters(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for mod in self.modules():
            if isinstance(mod, MSDeformAttn):
                mod._reset_parameters()
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

    def forward(self, srcs, masks, pos_embeds, query_embed=None, targets=None):
        assert query_embed is not None
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
        query_pos, tgt = torch.split(query_embed, c, dim=1)
        query_pos = query_pos.unsqueeze(0).expand(bs, -1, -1)
        tgt = tgt.unsqueeze(0).expand(bs, -1, -1)
        reference_points = self.reference_points(query_pos).sigmoid()
        padded_queries = None

        if targets is not None and "track_query_hs_embeds" in targets[0]:
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
        return hs, memory, init_reference, inter_references, refined, None


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
