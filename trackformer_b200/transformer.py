"""Vanilla DETR transformer (6 encoder + 6 decoder layers of dense multi-head attention) on the H100 kernels.

Mirror of src/trackformer/models/transformer.py: ``Transformer``, ``TransformerEncoder(Layer)``,
``TransformerDecoder(Layer)`` and ``build_transformer(args)`` with the same module and parameter names
(``encoder.layers.{i}.self_attn.in_proj_weight``, ``.linear1``, ``.norm1``, ``decoder.layers.{i}.multihead_attn.*``,
``decoder.norm``, ...), so the reference's checkpoints load by key.  Post-norm (``forward_post``, every shipped config)
and pre-norm (``forward_pre``, ``pre_norm: true``) layers; the decoder always returns its intermediate outputs as
``build_transformer`` asks.

On CUDA the three attention calls run on the dense-attention kernels (dense_attention.py; the decoder's query
self-attention on the small-attention kernels of small_attention.py, sized for it), the FFN on ``fused_linear`` /
``relu_dropout`` and the post-norm residuals on ``add_dropout_layernorm``; elsewhere on the stock modules.

``Transformer.forward`` takes one argument the reference does not: ``tgt_key_padding_mask`` [B, Q] (True = filler
query), the key padding of the decoder's query self-attention.  Filler track queries (fixed-shape CUDA-graph replays)
are hidden from the real queries as keys, and every other decoder op is row-wise, so the real rows are unaffected.
``track_attention=True`` (the reference's separate track-query self-attention, which hard-codes 100 object queries) is
not built.

``need_weights=True`` (``Transformer.forward``, ``TransformerDecoder.forward``) asks the LAST decoder layer's
cross-attention for its weights averaged over heads -- what the reference's tracker hooks out of
``decoder.layers[-1].multihead_attn`` for ``generate_attention_maps`` -- and ``Transformer.forward`` returns them as a
fourth value, ``[B, Q, h, w]`` on the memory grid.  Off (the default), nothing is computed and the return is unchanged.
"""
from __future__ import annotations

import copy

import torch
import torch.nn.functional as F
from torch import nn

from . import dense_attention, seeds, small_attention
from .fused_linear import linear as fused_linear, relu_dropout
from .fused_norm import add_dropout_layernorm


def _clones(module: nn.Module, n: int) -> nn.ModuleList:
    return nn.ModuleList([copy.deepcopy(module) for _ in range(n)])


def _activation(name: str):
    try:
        return {"relu": F.relu, "gelu": F.gelu, "glu": F.glu}[name]
    except KeyError:
        raise RuntimeError(f"activation should be relu/gelu, not {name}.") from None


def _add_pos(x, pos):
    return x if pos is None else x + pos


def _ffn(x, linear1, linear2, activation, dropout):
    a = fused_linear(x, linear1.weight, linear1.bias)
    h = relu_dropout(a, dropout) if activation is F.relu else dropout(activation(a))
    return fused_linear(h, linear2.weight, linear2.bias)


def _self_attention(module, qk, value, key_padding_mask):
    if small_attention.supported(module, qk):
        return small_attention.mha_forward(module, qk, value, key_padding_mask)
    return dense_attention.attention(module, qk, qk, value, key_padding_mask)


class Transformer(nn.Module):
    def __init__(self, d_model=512, nhead=8, num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=2048,
                 dropout=0.1, activation="relu", normalize_before=False, return_intermediate_dec=False,
                 track_attention=False):
        super().__init__()
        if track_attention:
            raise NotImplementedError("track_attention is not supported (no shipped config sets it)")
        encoder_layer = TransformerEncoderLayer(d_model, nhead, dim_feedforward, dropout, activation, normalize_before)
        encoder_norm = nn.LayerNorm(d_model) if normalize_before else None
        self.encoder = TransformerEncoder(encoder_layer, num_encoder_layers, encoder_norm)
        decoder_layer = TransformerDecoderLayer(d_model, nhead, dim_feedforward, dropout, activation, normalize_before)
        self.decoder = TransformerDecoder(decoder_layer, encoder_layer, num_decoder_layers, nn.LayerNorm(d_model),
                                          return_intermediate=return_intermediate_dec)
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        self.d_model = d_model
        self.nhead = nhead

    def forward(self, src, mask, query_embed, pos_embed, tgt=None, prev_frame=None, tgt_key_padding_mask=None,
                need_weights=False):
        """src [B, C, h, w], mask [B, h, w], query_embed [Q, B, C], pos_embed [B, C, h, w], tgt [Q, B, C] or None
        -> (hs [layers, B, Q, C], hs_without_norm [layers, B, Q, C], memory [B, C, h, w]), and with ``need_weights``
        the last decoder layer's head-averaged cross-attention weights [B, Q, h, w] as a fourth value."""
        if prev_frame is not None:
            raise NotImplementedError("prev_frame is only used by track_attention, which is not supported")
        if self.training and src.is_cuda:
            seeds.begin_step(src.device)          # one launch draws the dropout seeds of every fused site of this pass
        bs, c, h, w = src.shape
        src = src.flatten(2).permute(2, 0, 1).contiguous()
        pos_embed = pos_embed.flatten(2).permute(2, 0, 1).contiguous()
        mask = mask.flatten(1)
        if tgt is None:
            tgt = torch.zeros_like(query_embed)
        memory = self.encoder(src, src_key_padding_mask=mask, pos=pos_embed)
        dec = self.decoder(tgt, memory, tgt_key_padding_mask=tgt_key_padding_mask, memory_key_padding_mask=mask,
                           pos=pos_embed, query_pos=query_embed, need_weights=need_weights)
        hs, hs_without_norm = dec[0], dec[1]
        res = hs.transpose(1, 2), hs_without_norm.transpose(1, 2), memory.permute(1, 2, 0).view(bs, c, h, w)
        if need_weights:
            return res + (dec[2].view(bs, -1, h, w),)
        return res


class TransformerEncoder(nn.Module):
    def __init__(self, encoder_layer, num_layers, norm=None):
        super().__init__()
        self.layers = _clones(encoder_layer, num_layers)
        self.num_layers = num_layers
        self.norm = norm

    def forward(self, src, mask=None, src_key_padding_mask=None, pos=None):
        if mask is not None:
            raise NotImplementedError("attention masks other than key padding are not supported")
        output = src
        for layer in self.layers:
            output = layer(output, src_key_padding_mask=src_key_padding_mask, pos=pos)
        if self.norm is not None:
            output = self.norm(output)
        return output


class TransformerDecoder(nn.Module):
    def __init__(self, decoder_layer, encoder_layer, num_layers, norm=None, return_intermediate=False,
                 track_attention=False):
        """The reference's signature; ``encoder_layer`` only serves ``track_attention``, which is not supported."""
        super().__init__()
        if track_attention:
            raise NotImplementedError("track_attention is not supported (no shipped config sets it)")
        self.layers = _clones(decoder_layer, num_layers)
        self.num_layers = num_layers
        self.norm = norm
        self.return_intermediate = return_intermediate
        self.track_attention = False

    def forward(self, tgt, memory, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None,
                memory_key_padding_mask=None, pos=None, query_pos=None, need_weights=False):
        """-> (output, output without the final norm), plus the last layer's head-averaged cross-attention weights
        [B, Q, Lk] when ``need_weights``."""
        if tgt_mask is not None or memory_mask is not None:
            raise NotImplementedError("attention masks other than key padding are not supported")
        output = tgt
        intermediate = []
        for i, layer in enumerate(self.layers):
            output = layer(output, memory, tgt_key_padding_mask=tgt_key_padding_mask,
                           memory_key_padding_mask=memory_key_padding_mask, pos=pos, query_pos=query_pos,
                           need_weights=need_weights and i + 1 == len(self.layers))
            if need_weights and i + 1 == len(self.layers):
                output, weights = output
            if self.return_intermediate:
                intermediate.append(output)
        if self.return_intermediate:
            output = torch.stack(intermediate)
        res = (self.norm(output), output) if self.norm is not None else (output, output)
        return res + (weights,) if need_weights else res


class TransformerEncoderLayer(nn.Module):
    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", normalize_before=False):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)
        self.dropout1 = nn.Dropout(dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.activation = _activation(activation)
        self.normalize_before = normalize_before

    with_pos_embed = staticmethod(_add_pos)

    def forward_post(self, src, src_key_padding_mask=None, pos=None):
        qk = _add_pos(src, pos)
        src2 = dense_attention.attention(self.self_attn, qk, qk, src, src_key_padding_mask)
        src = add_dropout_layernorm(src, src2, self.dropout1, self.norm1)
        src2 = _ffn(src, self.linear1, self.linear2, self.activation, self.dropout)
        return add_dropout_layernorm(src, src2, self.dropout2, self.norm2)

    def forward_pre(self, src, src_key_padding_mask=None, pos=None):
        src2 = self.norm1(src)
        qk = _add_pos(src2, pos)
        src = src + self.dropout1(dense_attention.attention(self.self_attn, qk, qk, src2, src_key_padding_mask))
        src2 = _ffn(self.norm2(src), self.linear1, self.linear2, self.activation, self.dropout)
        return src + self.dropout2(src2)

    def forward(self, src, src_mask=None, src_key_padding_mask=None, pos=None):
        if src_mask is not None:
            raise NotImplementedError("attention masks other than key padding are not supported")
        if self.normalize_before:
            return self.forward_pre(src, src_key_padding_mask, pos)
        return self.forward_post(src, src_key_padding_mask, pos)


class TransformerDecoderLayer(nn.Module):
    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", normalize_before=False):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.multihead_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)
        self.norm3 = nn.LayerNorm(d_model)
        self.dropout1 = nn.Dropout(dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.dropout3 = nn.Dropout(dropout)
        self.activation = _activation(activation)
        self.normalize_before = normalize_before

    with_pos_embed = staticmethod(_add_pos)

    def forward_post(self, tgt, memory, tgt_key_padding_mask=None, memory_key_padding_mask=None, pos=None,
                     query_pos=None, need_weights=False):
        tgt2 = _self_attention(self.self_attn, _add_pos(tgt, query_pos), tgt, tgt_key_padding_mask)
        tgt = add_dropout_layernorm(tgt, tgt2, self.dropout1, self.norm1)
        tgt2 = dense_attention.attention(self.multihead_attn, _add_pos(tgt, query_pos), _add_pos(memory, pos), memory,
                                         memory_key_padding_mask, need_weights)
        if need_weights:
            tgt2, weights = tgt2
        tgt = add_dropout_layernorm(tgt, tgt2, self.dropout2, self.norm2)
        tgt2 = _ffn(tgt, self.linear1, self.linear2, self.activation, self.dropout)
        tgt = add_dropout_layernorm(tgt, tgt2, self.dropout3, self.norm3)
        return (tgt, weights) if need_weights else tgt

    def forward_pre(self, tgt, memory, tgt_key_padding_mask=None, memory_key_padding_mask=None, pos=None,
                    query_pos=None, need_weights=False):
        tgt2 = self.norm1(tgt)
        tgt = tgt + self.dropout1(_self_attention(self.self_attn, _add_pos(tgt2, query_pos), tgt2, tgt_key_padding_mask))
        tgt2 = self.norm2(tgt)
        tgt2 = dense_attention.attention(self.multihead_attn, _add_pos(tgt2, query_pos), _add_pos(memory, pos), memory,
                                         memory_key_padding_mask, need_weights)
        if need_weights:
            tgt2, weights = tgt2
        tgt = tgt + self.dropout2(tgt2)
        tgt2 = _ffn(self.norm3(tgt), self.linear1, self.linear2, self.activation, self.dropout)
        tgt = tgt + self.dropout3(tgt2)
        return (tgt, weights) if need_weights else tgt

    def forward(self, tgt, memory, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None,
                memory_key_padding_mask=None, pos=None, query_pos=None, need_weights=False):
        """-> tgt, or ``(tgt, cross-attention weights averaged over heads [B, Q, Lk])`` with ``need_weights``."""
        if tgt_mask is not None or memory_mask is not None:
            raise NotImplementedError("attention masks other than key padding are not supported")
        if self.normalize_before:
            return self.forward_pre(tgt, memory, tgt_key_padding_mask, memory_key_padding_mask, pos, query_pos,
                                    need_weights)
        return self.forward_post(tgt, memory, tgt_key_padding_mask, memory_key_padding_mask, pos, query_pos,
                                 need_weights)


def build_transformer(args):
    return Transformer(d_model=args.hidden_dim, dropout=args.dropout, nhead=args.nheads,
                       dim_feedforward=args.dim_feedforward, num_encoder_layers=args.enc_layers,
                       num_decoder_layers=args.dec_layers, normalize_before=args.pre_norm,
                       return_intermediate_dec=True, track_attention=args.track_attention)
