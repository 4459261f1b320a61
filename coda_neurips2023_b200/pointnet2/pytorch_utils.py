"""Shared 1x1-conv MLP blocks with the reference's module tree.

Mirrors the public names and, more importantly, the *parameter paths* of
third_party_pointnet2/pointnet2/pytorch_utils.py (``layer{i}.conv.weight``,
``layer{i}.bn.bn.{weight,bias,running_mean,running_var,num_batches_tracked}``) so
that checkpoints written by the reference load unchanged (SURVEY.md section 5).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F


class _NormWrap(nn.Sequential):
    """`bn` submodule holding a `bn` child: gives the `.bn.bn.weight` key path
    (reference pytorch_utils.py:36-44); affine initialised to (1, 0)."""

    def __init__(self, channels: int, norm_cls, name: str = ""):
        super().__init__()
        self.add_module(name + "bn", norm_cls(channels))
        nn.init.constant_(self[0].weight, 1.0)
        nn.init.constant_(self[0].bias, 0.0)


class BatchNorm1d(_NormWrap):
    def __init__(self, in_size: int, *, name: str = ""):
        super().__init__(in_size, nn.BatchNorm1d, name)


class BatchNorm2d(_NormWrap):
    def __init__(self, in_size: int, name: str = ""):
        super().__init__(in_size, nn.BatchNorm2d, name)


class BatchNorm3d(_NormWrap):
    def __init__(self, in_size: int, name: str = ""):
        super().__init__(in_size, nn.BatchNorm3d, name)


class _ConvBlock(nn.Sequential):
    """conv (+ bn) (+ activation), or pre-activation order; a conv bias exists
    only when there is no batch norm (reference pytorch_utils.py:65-118)."""

    _conv_cls = None
    _norm_cls = None
    _default_kernel: Sequence[int] | int = 1

    def __init__(self, in_size: int, out_size: int, *, kernel_size=None, stride=None, padding=None,
                 activation=nn.ReLU(inplace=True), bn: bool = False, init=nn.init.kaiming_normal_,
                 bias: bool = True, preact: bool = False, name: str = ""):
        super().__init__()
        nd = {nn.Conv1d: 1, nn.Conv2d: 2, nn.Conv3d: 3}[self._conv_cls]
        if kernel_size is None:
            kernel_size = 1 if nd == 1 else (1,) * nd
        if stride is None:
            stride = 1 if nd == 1 else (1,) * nd
        if padding is None:
            padding = 0 if nd == 1 else (0,) * nd
        conv = self._conv_cls(in_size, out_size, kernel_size=kernel_size, stride=stride,
                              padding=padding, bias=bias and not bn)
        init(conv.weight)
        if conv.bias is not None:
            nn.init.constant_(conv.bias, 0.0)
        norm = self._norm_cls(in_size if preact else out_size) if bn else None
        tail = []
        if norm is not None:
            tail.append((name + "bn", norm))
        if activation is not None:
            tail.append((name + "activation", activation))
        order = tail + [(name + "conv", conv)] if preact else [(name + "conv", conv)] + tail
        for key, mod in order:
            self.add_module(key, mod)


class Conv1d(_ConvBlock):
    _conv_cls = nn.Conv1d
    _norm_cls = BatchNorm1d


class Conv2d(_ConvBlock):
    _conv_cls = nn.Conv2d
    _norm_cls = BatchNorm2d


class Conv3d(_ConvBlock):
    _conv_cls = nn.Conv3d
    _norm_cls = BatchNorm3d


def _batch_norm_rows(bn: nn.modules.batchnorm._BatchNorm, h: torch.Tensor) -> torch.Tensor:
    """BatchNorm{1,2,3}d semantics (train-mode batch statistics, running-stat update) on a
    channels-last (rows, C) tensor."""
    momentum = 0.0 if bn.momentum is None else bn.momentum
    if bn.training and bn.track_running_stats and bn.num_batches_tracked is not None:
        bn.num_batches_tracked.add_(1)
        if bn.momentum is None:
            momentum = 1.0 / float(bn.num_batches_tracked)
    use_batch = bn.training or (bn.running_mean is None and bn.running_var is None)
    return F.batch_norm(h, bn.running_mean if (not bn.training or bn.track_running_stats) else None,
                        bn.running_var if (not bn.training or bn.track_running_stats) else None,
                        bn.weight, bn.bias, use_batch, momentum, bn.eps)


def _is_bn2d(slot) -> bool:
    """Does a block's `_NormWrap` slot hold a 2-D BatchNorm: an nn.BatchNorm2d, or the nn.SyncBatchNorm that
    convert_sync_batchnorm put in its place?  A SyncBatchNorm has no dimensionality of its own: the slot (this
    module's BatchNorm2d wrapper) gives it."""
    return isinstance(slot, _NormWrap) and (isinstance(slot[0], nn.BatchNorm2d)
                                            or (isinstance(slot, BatchNorm2d) and isinstance(slot[0], nn.SyncBatchNorm)))


class SharedMLP(nn.Sequential):
    """Stack of 1x1 Conv2d blocks: `layer0`, `layer1`, ... (reference
    pytorch_utils.py:8-33).  Executed channels-last: the (B, C, npoint, nsample) map is
    (B*npoint*nsample, C) rows, each block one wgmma GEMM + BatchNorm over rows + ReLU."""

    def forward(self, x):
        from .. import ops

        if x.dim() != 4 or not x.is_cuda:
            return super().forward(x)
        b, c, p, s = x.shape
        h = x.permute(0, 2, 3, 1).reshape(b * p * s, c)
        for block in self:
            for name, mod in block.named_children():
                if isinstance(mod, nn.Conv2d):
                    if mod.kernel_size != (1, 1):
                        norms = [m[0] for m in self.modules() if isinstance(m, _NormWrap)]
                        if any(ops.bn_sync_group(bn) is not None for bn in norms):
                            raise NotImplementedError("synchronised BatchNorm after a convolution wider than 1x1")
                        return super().forward(x)
                    h = ops.linear(h, mod.weight.reshape(mod.weight.shape[0], -1), mod.bias)
                elif isinstance(mod, _NormWrap):
                    if ops.bn_sync_group(mod[0]) is not None:
                        # synchronised statistics over every rank's rows (or NotImplementedError), never per-GPU ones
                        h = ops.bn_act_rows(h, mod[0], relu=False, drop_p=0.0, training=True)
                    else:
                        h = _batch_norm_rows(mod[0], h)
                elif isinstance(mod, nn.ReLU):
                    h = torch.relu(h)
                else:
                    h = mod(h)
        return h.view(b, p, s, -1).permute(0, 3, 1, 2)

    def forward_max_pooled(self, x):
        """relu(bn(conv(.))) blocks followed by the max over the last (nsample) axis, as one fused autograd
        node (sa_mlp.shared_mlp_max): (B, C, npoint, nsample) -> (B, C_out, npoint).  Returns None when the
        fused path does not apply (CPU, eval mode, other block layouts); the caller then runs forward() and
        pools itself.  The BatchNorm of a block may be the nn.SyncBatchNorm convert_sync_batchnorm made of it
        (the `_NormWrap` slot says it is 2-D); the node synchronises it as ops.bn_sync_group says."""
        from .. import sa_mlp

        if x.dim() != 4 or not x.is_cuda or not torch.is_grad_enabled():
            return None
        blocks = []
        for block in self:
            mods = list(block.children())
            if (len(mods) != 3 or not isinstance(mods[0], nn.Conv2d) or mods[0].kernel_size != (1, 1)
                    or not _is_bn2d(mods[1]) or not isinstance(mods[2], nn.ReLU)):
                return None
            blocks.append((mods[0], mods[1][0]))
        b, c, p, s = x.shape
        rows = x.permute(0, 2, 3, 1).reshape(b * p * s, c)
        if not sa_mlp.applicable(rows, blocks, s):
            return None
        pooled = sa_mlp.shared_mlp_max(rows, blocks, s)          # (B * npoint, C_out)
        return pooled.view(b, p, -1).permute(0, 2, 1)

    def forward_max_pooled_infer(self, x):
        """Inference form of forward_max_pooled (eval-mode BatchNorm with running statistics, nothing for autograd
        to record): the whole MLP + max over nsample as one kernel (sa_mlp.shared_mlp_max_infer) that reads the
        grouped (B, C, npoint, nsample) map in place -> (B, C_out, npoint).  Returns None when it does not apply
        (training-mode BatchNorm, gradients wanted, a layout other than the pre-encoder's); the caller then runs
        forward() and pools itself."""
        from .. import sa_mlp

        if x.dim() != 4 or not x.is_cuda:
            return None
        blocks = []
        for block in self:
            mods = list(block.children())
            if (len(mods) != 3 or not isinstance(mods[0], nn.Conv2d) or mods[0].kernel_size != (1, 1)
                    or not _is_bn2d(mods[1]) or not isinstance(mods[2], nn.ReLU)):
                return None
            blocks.append((mods[0], mods[1][0]))
        b, _, p, s = x.shape
        if not sa_mlp.infer_applicable(x, blocks, s):
            return None
        pooled = sa_mlp.shared_mlp_max_infer(x, blocks, s)       # (B * npoint, C_out)
        return pooled.view(b, p, -1).permute(0, 2, 1)

    def __init__(self, args: List[int], *, bn: bool = False, activation=nn.ReLU(inplace=True),
                 preact: bool = False, first: bool = False, name: str = ""):
        super().__init__()
        for i in range(len(args) - 1):
            plain = first and preact and i == 0  # the very first pre-act block has no bn/act
            self.add_module(
                f"{name}layer{i}",
                Conv2d(args[i], args[i + 1], bn=bn and not plain,
                       activation=None if plain else activation, preact=preact))


class FC(nn.Sequential):
    """Linear (+ BatchNorm1d) (+ activation) (reference pytorch_utils.py:219-254)."""

    def __init__(self, in_size: int, out_size: int, *, activation=nn.ReLU(inplace=True),
                 bn: bool = False, init=None, preact: bool = False, name: str = ""):
        super().__init__()
        fc = nn.Linear(in_size, out_size, bias=not bn)
        if init is not None:
            init(fc.weight)
        if not bn:
            nn.init.constant_(fc.bias, 0.0)
        tail = []
        if bn:
            tail.append((name + "bn", BatchNorm1d(in_size if preact else out_size)))
        if activation is not None:
            tail.append((name + "activation", activation))
        order = tail + [(name + "fc", fc)] if preact else [(name + "fc", fc)] + tail
        for key, mod in order:
            self.add_module(key, mod)


def set_bn_momentum_default(bn_momentum):
    def fn(m):
        if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d)):
            m.momentum = bn_momentum
    return fn


class BNMomentumScheduler:
    """Applies `bn_lambda(epoch)` as the momentum of every BatchNorm in `model`."""

    def __init__(self, model, bn_lambda, last_epoch: int = -1, setter=set_bn_momentum_default):
        if not isinstance(model, nn.Module):
            raise RuntimeError(f"Class '{type(model).__name__}' is not a PyTorch nn Module")
        self.model, self.setter, self.lmbd = model, setter, bn_lambda
        self.step(last_epoch + 1)
        self.last_epoch = last_epoch

    def step(self, epoch: Optional[int] = None):
        if epoch is None:
            epoch = self.last_epoch + 1
        self.last_epoch = epoch
        self.model.apply(self.setter(self.lmbd(epoch)))
