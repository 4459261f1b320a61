"""3DETR transformer encoder / decoder (mirror of the LIVE classes of reference
models/transformer.py: TransformerEncoder, TransformerEncoderLayer,
MaskedTransformerEncoder, TransformerDecoder, TransformerDecoderLayer).

Differences from the reference are implementation-only: attention runs in the
fused wgmma kernel (no (B*H, L, L) probability tensor is written, no head
averaging), LayerNorm is the warp-per-row kernel, and the K/V input projections
of one packed weight are issued as single GEMMs.  Parameter names and shapes
match `nn.MultiheadAttention` / the reference layers so checkpoints interchange.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import Tensor, nn

from .. import ops
from .helpers import ACTIVATION_DICT, NORM_DICT, WEIGHT_INIT_DICT, get_clones


class MultiheadAttention(nn.Module):
    """Drop-in for `nn.MultiheadAttention(embed_dim, num_heads, dropout)` as the
    reference uses it (sequence-first, packed in_proj, bias, no kdim/vdim).

    forward(query, key, value, attn_mask=None, key_padding_mask=None) -> (out, None);
    attention weights are not returned (the reference discards them everywhere
    except under `return_attn_weights`, which no shipped configuration sets).

    attn_mask: boolean (True = not visible), (Lq, Lk), (B, Lq, Lk) or the head-tiled (B*H, Lq, Lk) the reference's
    MaskedTransformerEncoder builds (every head carries the same mask: the first of each H is used) -- or the packed
    (bits_q, bits_k) pair of ops.attention_mask_bits / ops.radius_mask_bits, which skips the dense mask entirely.
    key_padding_mask (B, Lk) is folded into the same packed mask.
    """

    def __init__(self, embed_dim: int, num_heads: int, dropout: float = 0.0):
        super().__init__()
        assert embed_dim % num_heads == 0
        self.embed_dim, self.num_heads, self.dropout = embed_dim, num_heads, dropout
        self.head_dim = embed_dim // num_heads
        self.in_proj_weight = nn.Parameter(torch.empty(3 * embed_dim, embed_dim))
        self.in_proj_bias = nn.Parameter(torch.empty(3 * embed_dim))
        self.out_proj = ops.Linear(embed_dim, embed_dim, bias=True)
        self._reset_parameters()

    def _reset_parameters(self):
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.constant_(self.in_proj_bias, 0.0)
        nn.init.constant_(self.out_proj.bias, 0.0)

    def forward(self, query: Tensor, key: Tensor, value: Tensor, attn_mask: Optional[Tensor] = None,
                key_padding_mask: Optional[Tensor] = None, need_weights: bool = False):
        e = self.embed_dim
        w, b = self.in_proj_weight, self.in_proj_bias
        mask = self._packed_mask(attn_mask, key_padding_mask, query.shape[1], query.shape[0], key.shape[0])
        if query is key and key is value:      # encoder self-attention: ONE fused q|k|v GEMM, consumed in place
            out = ops.attention_fused(ops.linear(query, w, b), None, "qkv", self.num_heads, self.dropout,
                                      self.training, mask)
        elif query is key:                      # decoder self-attention: q = k = tgt + pos (fused q|k GEMM), v = tgt
            out = ops.attention_fused(ops.linear(query, w[: 2 * e], b[: 2 * e]), ops.linear(value, w[2 * e:], b[2 * e:]),
                                      "qk_v", self.num_heads, self.dropout, self.training, mask)
        else:                                   # cross-attention
            q = ops.linear(query, w[:e], b[:e])
            k = ops.linear(key, w[e: 2 * e], b[e: 2 * e])
            v = ops.linear(value, w[2 * e:], b[2 * e:])
            out = ops.attention(q, k, v, self.num_heads, self.dropout, self.training, mask=mask)
        return self.out_proj(out), None

    def forward_bank(self, query: Tensor, bank, token, idx: int):
        """cross-attention whose keys / values were projected for all layers at once (ops.KVBank)"""
        e = self.embed_dim
        q = ops.linear(query, self.in_proj_weight[:e], self.in_proj_bias[:e])
        out = ops.attention_bank(q, bank, token, idx, self.num_heads, self.dropout, self.training)
        return self.out_proj(out), None

    def _packed_mask(self, attn_mask, key_padding_mask, batch, lq, lk):
        if attn_mask is None and key_padding_mask is None:
            return None
        if isinstance(attn_mask, tuple):          # already packed
            if key_padding_mask is not None:
                raise NotImplementedError("key_padding_mask together with a pre-packed attn_mask")
            return attn_mask
        m = None
        if attn_mask is not None:
            if attn_mask.dtype != torch.bool:
                if attn_mask.is_floating_point():
                    raise NotImplementedError("additive float attention masks: pass a boolean mask")
                attn_mask = attn_mask != 0
            m = attn_mask
            if m.dim() == 3 and m.shape[0] == batch * self.num_heads and self.num_heads > 1:
                m = m[:: self.num_heads]         # head-tiled copy of a per-scene mask (reference transformer.py:190-194)
            if m.dim() == 2:
                m = m.unsqueeze(0)
        if key_padding_mask is not None:
            kp = key_padding_mask.to(torch.bool).view(batch, 1, lk)
            m = kp.expand(batch, lq, lk) if m is None else (m | kp)
        return ops.attention_mask_bits(m, batch)


class TransformerEncoder(nn.Module):
    def __init__(self, encoder_layer, num_layers, norm=None, weight_init_name="xavier_uniform"):
        super().__init__()
        self.layers = get_clones(encoder_layer, num_layers)
        self.num_layers = num_layers
        self.norm = norm
        self._reset_parameters(weight_init_name)

    def _reset_parameters(self, weight_init_name):
        func = WEIGHT_INIT_DICT[weight_init_name]
        for p in self.parameters():
            if p.dim() > 1:
                func(p)

    def forward(self, src, mask: Optional[Tensor] = None, src_key_padding_mask: Optional[Tensor] = None,
                pos: Optional[Tensor] = None, xyz: Optional[Tensor] = None, transpose_swap: Optional[bool] = False):
        """src (L, B, C) -> (xyz, output (L, B, C), None)   [reference transformer.py:35-74]"""
        if transpose_swap:
            bs, c, h, w = src.shape
            src = src.flatten(2).permute(2, 0, 1)
            if pos is not None:
                pos = pos.flatten(2).permute(2, 0, 1)
        output = src
        for layer in self.layers:
            output = layer(output, src_mask=mask, src_key_padding_mask=src_key_padding_mask, pos=pos)
        if self.norm is not None:
            output = self.norm(output)
        if transpose_swap:
            output = output.permute(1, 2, 0).view(bs, c, h, w).contiguous()
        return xyz, output, None


class MaskedTransformerEncoder(TransformerEncoder):
    """`--enc_type masked` (reference models/transformer.py:146-211): layer l only attends within
    `masking_radius[l]` of each point; after the first layer the points are down-sampled by a set-abstraction
    module.  The radius mask is built bit-packed on the device straight from the coordinates (no (B, N, N) distance
    matrix, no head-tiled copy) and applied inside the fused attention kernels, forward and backward."""

    def __init__(self, encoder_layer, num_layers, masking_radius, interim_downsampling, norm=None,
                 weight_init_name="xavier_uniform"):
        super().__init__(encoder_layer, num_layers, norm=norm, weight_init_name=weight_init_name)
        assert len(masking_radius) == num_layers
        self.masking_radius = masking_radius
        self.interim_downsampling = interim_downsampling

    def compute_mask(self, xyz, radius, dist=None):
        """The reference's dense form (boolean (B, N, N), True = outside the radius) -- kept for callers / tests; the
        forward below uses the packed form."""
        with torch.no_grad():
            if dist is None or dist.shape[1] != xyz.shape[1]:
                dist = torch.cdist(xyz, xyz, p=2)
            return dist >= radius, dist

    def forward(self, src, mask: Optional[Tensor] = None, src_key_padding_mask: Optional[Tensor] = None,
                pos: Optional[Tensor] = None, xyz: Optional[Tensor] = None, transpose_swap: Optional[bool] = False):
        if transpose_swap:
            bs, c, h, w = src.shape
            src = src.flatten(2).permute(2, 0, 1)
            if pos is not None:
                pos = pos.flatten(2).permute(2, 0, 1)
        output = src
        xyz_inds = None
        for idx, layer in enumerate(self.layers):
            lmask = None
            if self.masking_radius[idx] > 0:
                lmask = ops.radius_mask_bits(xyz, self.masking_radius[idx])
            output = layer(output, src_mask=lmask, src_key_padding_mask=src_key_padding_mask, pos=pos)
            if idx == 0 and self.interim_downsampling:
                # (npoints, batch, channel) -> (batch, channel, npoints) for the set-abstraction module and back
                xyz, output, xyz_inds = self.interim_downsampling(xyz, output.permute(1, 2, 0).contiguous())
                output = output.permute(2, 0, 1)
        if self.norm is not None:
            output = self.norm(output)
        if transpose_swap:
            output = output.permute(1, 2, 0).view(bs, c, h, w).contiguous()
        return xyz, output, xyz_inds

    def extra_repr(self):
        return "masking_radius=" + ", ".join("%.2f" % x for x in self.masking_radius)


class TransformerEncoderLayer(nn.Module):
    def __init__(self, d_model, nhead=4, dim_feedforward=128, dropout=0.1, dropout_attn=None,
                 activation="relu", normalize_before=True, norm_name="ln", use_ffn=True, ffn_use_bias=True):
        super().__init__()
        if dropout_attn is None:
            dropout_attn = dropout
        self.self_attn = MultiheadAttention(d_model, nhead, dropout=dropout_attn)
        self.use_ffn = use_ffn
        if self.use_ffn:
            self.linear1 = ops.Linear(d_model, dim_feedforward, bias=ffn_use_bias)
            self.dropout = nn.Dropout(dropout, inplace=False)
            self.linear2 = ops.Linear(dim_feedforward, d_model, bias=ffn_use_bias)
            self.norm2 = NORM_DICT[norm_name](d_model)
            self.dropout2 = nn.Dropout(dropout, inplace=False)
        self.norm1 = NORM_DICT[norm_name](d_model)
        self.dropout1 = nn.Dropout(dropout, inplace=False)
        self.activation = ACTIVATION_DICT[activation]()
        self.normalize_before = normalize_before
        self.nhead = nhead

    @staticmethod
    def with_pos_embed(tensor, pos: Optional[Tensor]):
        return tensor if pos is None else tensor + pos

    def forward_pre(self, src, src_mask=None, src_key_padding_mask=None, pos=None, return_attn_weights=False):
        # reference transformer.py:461-479
        # norm -> (residual operand, norm(src), norm(src) + pos) as one node: the joins of the residual branch and of
        # the `+ pos` branch happen inside the LayerNorm kernels (ops.layer_norm_branch)
        src, src2, qk = ops.layer_norm_branch(src, self.norm1, pos)
        attn = self.self_attn(qk, qk, src2, attn_mask=src_mask, key_padding_mask=src_key_padding_mask)[0]
        src = ops.dropout_add(attn, src, self.dropout1.p, self.training)
        if self.use_ffn:
            src, src2, _ = ops.layer_norm_branch(src, self.norm2)
            src2 = self.linear2(ops.dropout(_ffn_hidden(self, src2), self.dropout.p, self.training))
            src = ops.dropout_add(src2, src, self.dropout2.p, self.training)
        if return_attn_weights:
            return src, None
        return src

    def forward_post(self, src, src_mask=None, src_key_padding_mask=None, pos=None):
        qk = self.with_pos_embed(src, pos)
        src2 = self.self_attn(qk, qk, src, attn_mask=src_mask, key_padding_mask=src_key_padding_mask)[0]
        src = self.norm1(ops.dropout_add(src2, src, self.dropout1.p, self.training))
        if self.use_ffn:
            src2 = self.linear2(ops.dropout(_ffn_hidden(self, src), self.dropout.p, self.training))
            src = self.norm2(ops.dropout_add(src2, src, self.dropout2.p, self.training))
        return src

    def forward(self, src, src_mask=None, src_key_padding_mask=None, pos=None, return_attn_weights=False):
        if self.normalize_before:
            return self.forward_pre(src, src_mask, src_key_padding_mask, pos, return_attn_weights)
        return self.forward_post(src, src_mask, src_key_padding_mask, pos)

    def extra_repr(self):
        return f"attn_dr={self.self_attn.dropout}"


class TransformerDecoder(nn.Module):
    def __init__(self, decoder_layer, num_layers, norm_fn_name="ln", return_intermediate=False,
                 weight_init_name="xavier_uniform"):
        super().__init__()
        self.layers = get_clones(decoder_layer, num_layers)
        self.num_layers = num_layers
        self.norm = None
        if norm_fn_name is not None:
            self.norm = NORM_DICT[norm_fn_name](self.layers[0].linear2.out_features)
        self.return_intermediate = return_intermediate
        self._reset_parameters(weight_init_name)

    def _reset_parameters(self, weight_init_name):
        func = WEIGHT_INIT_DICT[weight_init_name]
        for p in self.parameters():
            if p.dim() > 1:
                func(p)

    def forward(self, tgt, memory, image_features_clip=None, text_features_clip=None, tgt_mask=None,
                memory_mask=None, tgt_key_padding_mask=None, memory_key_padding_mask=None,
                pos: Optional[Tensor] = None, query_pos: Optional[Tensor] = None,
                transpose_swap: Optional[bool] = False, return_attn_weights: Optional[bool] = False):
        """tgt (Q, B, C), memory (L, B, C) -> (stack of per-layer normed outputs (nl, Q, B, C), attns)
        [reference transformer.py:97-143]"""
        if transpose_swap:
            bs, c, h, w = memory.shape
            memory = memory.flatten(2).permute(2, 0, 1)
            if pos is not None:
                pos = pos.flatten(2).permute(2, 0, 1)
        if return_attn_weights:
            raise NotImplementedError("attention weights are not materialised by the fused kernel")
        # key of every cross-attention is memory + pos: formed once, not once per layer
        mem_key = memory if pos is None else memory + pos
        # ... and so are the K / V projections of all layers: two GEMMs instead of 2 x num_layers (ops.KVBank)
        kv = None
        cross = [layer.multihead_attn for layer in self.layers]
        if memory_mask is None and memory_key_padding_mask is None and ops.kv_bank_applicable(memory, cross):
            kv = ops.kv_bank(mem_key, memory, cross)
        output = tgt
        intermediate = []
        # every layer adds the query embedding twice (self- and cross-attention): its 2 x num_layers gradient
        # contributions meet in one n-ary sum (ops.fanout) instead of a chain of binary adds
        if query_pos is not None and not query_pos.is_contiguous():
            query_pos = query_pos.contiguous()      # once, not once per use inside the fused norm kernels
        qp = None if query_pos is None else ops.fanout(query_pos, 2 * len(self.layers))
        stacked = self.return_intermediate and self.norm is not None
        outputs = []
        for idx, layer in enumerate(self.layers):
            output, _ = layer(output, memory, tgt_mask=tgt_mask, memory_mask=memory_mask,
                              tgt_key_padding_mask=tgt_key_padding_mask,
                              memory_key_padding_mask=memory_key_padding_mask, pos=pos,
                              query_pos=None if qp is None else qp[2 * idx],
                              memory_key=mem_key, kv_bank=None if kv is None else (kv[0], kv[1], idx),
                              query_pos_cross=None if qp is None else qp[2 * idx + 1])
            if stacked:
                outputs.append(output)
            elif self.return_intermediate:
                intermediate.append(self.norm(output))
        if stacked and ops.norm_stack_applicable(self.norm, outputs):
            # (layers, batch, query, channel) buffer, returned as the reference's (layers, query, batch, channel)
            # view of it: the prediction heads' permute + reshape (models/model_3detr.py get_box_predictions) is free
            return ops.norm_stack(self.norm, outputs).permute(0, 2, 1, 3), []
        if stacked:
            intermediate = [self.norm(o) for o in outputs]
            return torch.stack(intermediate), []
        if self.norm is not None:
            output = self.norm(output)
            if self.return_intermediate:
                intermediate.pop()
                intermediate.append(output)
        if self.return_intermediate:
            return torch.stack(intermediate), []
        return output, []


def _ffn_hidden(layer, x):
    """activation(linear1(x)); with a ReLU activation the rectifier runs in the GEMM epilogue (one kernel less
    forward and backward)."""
    if isinstance(layer.activation, nn.ReLU):
        return ops.linear(x, layer.linear1.weight, layer.linear1.bias, relu=True)
    return layer.activation(layer.linear1(x))


class TransformerDecoderLayer(nn.Module):
    def __init__(self, d_model, nhead=4, dim_feedforward=256, dropout=0.1, dropout_attn=None,
                 activation="relu", normalize_before=True, norm_fn_name="ln"):
        super().__init__()
        self.self_attn = MultiheadAttention(d_model, nhead, dropout=dropout)
        self.multihead_attn = MultiheadAttention(d_model, nhead, dropout=dropout)
        self.norm1 = NORM_DICT[norm_fn_name](d_model)
        self.norm2 = NORM_DICT[norm_fn_name](d_model)
        self.norm3 = NORM_DICT[norm_fn_name](d_model)
        self.dropout1 = nn.Dropout(dropout, inplace=False)
        self.dropout2 = nn.Dropout(dropout, inplace=False)
        self.dropout3 = nn.Dropout(dropout, inplace=False)
        self.linear1 = ops.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout, inplace=False)
        self.linear2 = ops.Linear(dim_feedforward, d_model)
        self.activation = ACTIVATION_DICT[activation]()
        self.normalize_before = normalize_before

    @staticmethod
    def with_pos_embed(tensor, pos: Optional[Tensor]):
        return tensor if pos is None else tensor + pos

    def _cross(self, query, memory_key, memory, memory_mask, memory_key_padding_mask, kv_bank):
        if kv_bank is not None:
            return self.multihead_attn.forward_bank(query, *kv_bank)[0]
        return self.multihead_attn(query, memory_key, memory, attn_mask=memory_mask,
                                   key_padding_mask=memory_key_padding_mask)[0]

    def forward_pre(self, tgt, memory, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None,
                    memory_key_padding_mask=None, pos=None, query_pos=None, return_attn_weights=False,
                    memory_key=None, kv_bank=None, query_pos_cross=None):
        # reference transformer.py:556-580
        if memory_key is None:
            memory_key = self.with_pos_embed(memory, pos)
        if query_pos_cross is None:
            query_pos_cross = query_pos
        # each norm is one node with the residual by-pass and the `+ query_pos` operand (ops.layer_norm_branch)
        tgt, tgt2, qk = ops.layer_norm_branch(tgt, self.norm1, query_pos)
        tgt2 = self.self_attn(qk, qk, tgt2, attn_mask=tgt_mask, key_padding_mask=tgt_key_padding_mask)[0]
        tgt = ops.dropout_add(tgt2, tgt, self.dropout1.p, self.training)
        tgt, _, q = ops.layer_norm_branch(tgt, self.norm2, query_pos_cross, want_y=False)
        tgt2 = self._cross(q, memory_key, memory, memory_mask, memory_key_padding_mask, kv_bank)
        tgt = ops.dropout_add(tgt2, tgt, self.dropout2.p, self.training)
        tgt, tgt2, _ = ops.layer_norm_branch(tgt, self.norm3)
        tgt2 = self.linear2(ops.dropout(_ffn_hidden(self, tgt2), self.dropout.p, self.training))
        tgt = ops.dropout_add(tgt2, tgt, self.dropout3.p, self.training)
        return tgt, None

    def forward_post(self, tgt, memory, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None,
                     memory_key_padding_mask=None, pos=None, query_pos=None, return_attn_weights=False,
                     memory_key=None, kv_bank=None, query_pos_cross=None):
        if memory_key is None:
            memory_key = self.with_pos_embed(memory, pos)
        if query_pos_cross is None:
            query_pos_cross = query_pos
        qk = self.with_pos_embed(tgt, query_pos)
        tgt2 = self.self_attn(qk, qk, tgt, attn_mask=tgt_mask, key_padding_mask=tgt_key_padding_mask)[0]
        tgt = self.norm1(ops.dropout_add(tgt2, tgt, self.dropout1.p, self.training))
        tgt2 = self._cross(self.with_pos_embed(tgt, query_pos_cross), memory_key, memory, memory_mask,
                           memory_key_padding_mask, kv_bank)
        tgt = self.norm2(ops.dropout_add(tgt2, tgt, self.dropout2.p, self.training))
        tgt2 = self.linear2(ops.dropout(_ffn_hidden(self, tgt), self.dropout.p, self.training))
        tgt = self.norm3(ops.dropout_add(tgt2, tgt, self.dropout3.p, self.training))
        return tgt, None

    def forward(self, tgt, memory, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None,
                memory_key_padding_mask=None, pos=None, query_pos=None, return_attn_weights=False,
                memory_key=None, kv_bank=None, query_pos_cross=None):
        fn = self.forward_pre if self.normalize_before else self.forward_post
        return fn(tgt, memory, tgt_mask, memory_mask, tgt_key_padding_mask, memory_key_padding_mask, pos,
                  query_pos, return_attn_weights, memory_key, kv_bank, query_pos_cross)
