"""Building blocks shared by the 3DETR modules (mirror of reference models/helpers.py).

`NORM_DICT["ln"]` is the warp-per-row LayerNorm kernel (same parameters as nn.LayerNorm);
GenericMLP keeps the reference's nn.Module tree (parameter paths `layers.{i}`) but executes on
channels-last rows: wgmma GEMMs + one fused BatchNorm/ReLU/Dropout pass per block.
"""
from __future__ import annotations

import copy
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..ops import LayerNorm


class BatchNormDim1Swap(nn.BatchNorm1d):
    """BatchNorm1d for sequence-first (HW, N, C) tensors (reference helpers.py:8-24)."""

    def forward(self, x):
        return super().forward(x.permute(1, 2, 0)).permute(2, 0, 1)


NORM_DICT = {
    "bn": BatchNormDim1Swap,
    "bn1d": nn.BatchNorm1d,
    "id": nn.Identity,
    "ln": LayerNorm,
}

ACTIVATION_DICT = {
    "relu": nn.ReLU,
    "gelu": nn.GELU,
    "leakyrelu": partial(nn.LeakyReLU, negative_slope=0.1),
}

WEIGHT_INIT_DICT = {
    "xavier_uniform": nn.init.xavier_uniform_,
}


class GenericMLP(nn.Module):
    """[Conv1d|Linear -> norm -> act -> dropout] x len(hidden_dims) -> output layer.

    Same constructor arguments and `layers.{i}` parameter paths as reference
    models/helpers.py:45-112.
    """

    def __init__(self, input_dim, hidden_dims, output_dim, norm_fn_name=None, activation="relu",
                 use_conv=False, dropout=None, hidden_use_bias=False, output_use_bias=True,
                 output_use_activation=False, output_use_norm=False, weight_init_name=None):
        super().__init__()
        act = ACTIVATION_DICT[activation]
        norm = NORM_DICT[norm_fn_name] if norm_fn_name is not None else None
        if norm_fn_name == "ln" and use_conv:
            norm = lambda x: nn.GroupNorm(1, x)  # noqa: E731  LayerNorm over channels of a conv map
        if dropout is not None and not isinstance(dropout, list):
            dropout = [dropout for _ in range(len(hidden_dims))]

        def dense(i, o, bias):
            return nn.Conv1d(i, o, 1, bias=bias) if use_conv else nn.Linear(i, o, bias=bias)

        layers = []
        prev = input_dim
        for idx, width in enumerate(hidden_dims):
            layers.append(dense(prev, width, hidden_use_bias))
            if norm:
                layers.append(norm(width))
            layers.append(act())
            if dropout is not None:
                layers.append(nn.Dropout(p=dropout[idx]))
            prev = width
        layers.append(dense(prev, output_dim, output_use_bias))
        if output_use_norm:
            layers.append(norm(output_dim))
        if output_use_activation:
            layers.append(act())
        self.layers = nn.Sequential(*layers)
        if weight_init_name is not None:
            self.do_weight_init(weight_init_name)

    def do_weight_init(self, weight_init_name):
        func = WEIGHT_INIT_DICT[weight_init_name]
        for _, param in self.named_parameters():
            if param.dim() > 1:  # skips the norm layers
                func(param)

    def forward_rows(self, h):
        """The stack on channels-last rows (N, C_in) -> (N, C_out).  The 1x1 convolutions are GEMMs over the
        channel dim (ops.linear, wgmma); a [BatchNorm1d, ReLU, Dropout] run after a dense layer is ONE fused
        pass over the rows (ops.bn_act_rows: batch statistics, normalise + ReLU + counter-based dropout); a ReLU
        directly after a dense layer runs in the GEMM epilogue."""
        mods = list(self.layers)
        i = 0
        while i < len(mods):
            mod = mods[i]
            if isinstance(mod, (nn.Conv1d, nn.Linear)):
                fuse = i + 1 < len(mods) and isinstance(mods[i + 1], nn.ReLU)
                h = ops.linear(h, mod.weight.reshape(mod.weight.shape[0], -1), mod.bias, relu=fuse)
                i += 2 if fuse else 1
            elif isinstance(mod, nn.modules.batchnorm._BatchNorm):
                j = i + 1
                relu = j < len(mods) and isinstance(mods[j], nn.ReLU)
                j += 1 if relu else 0
                has_drop = j < len(mods) and isinstance(mods[j], nn.Dropout)
                drop = mods[j].p if has_drop else 0.0
                j += 1 if has_drop else 0
                h = ops.bn_act_rows(h, mod, relu, drop, self.training)
                i = j
            elif isinstance(mod, nn.Dropout):
                h = ops.dropout(h, mod.p, self.training)
                i += 1
            elif isinstance(mod, nn.GroupNorm):
                raise NotImplementedError("GroupNorm ('ln' on a conv MLP) is not used on the CoDA path")
            else:                                  # ReLU after a norm-less dense layer, LayerNorm
                h = mod(h)
                i += 1
        return h

    def forward(self, x):
        """(B, C, L) for the conv variant, (..., C) for the linear one."""
        if isinstance(self.layers[0], nn.Conv1d):
            b, c, l = x.shape
            h = self.forward_rows(x.transpose(1, 2).reshape(b * l, c))
            return h.view(b, l, -1).transpose(1, 2)
        lead = x.shape[:-1]
        return self.forward_rows(x.reshape(-1, x.shape[-1])).view(*lead, -1)


def get_clones(module, N):
    return nn.ModuleList([copy.deepcopy(module) for _ in range(N)])
