"""PointNet++ set-abstraction / feature-propagation modules.

Same class names, constructor keywords, forward signatures and parameter paths
as third_party_pointnet2/pointnet2/pointnet2_modules.py.  The model only builds
`PointnetSAModuleVotes` (models/model_3detr.py:12, :3935-3944); the other
classes are provided so that code importing them keeps working.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import pointnet2_utils
from . import pytorch_utils as pt_utils


def _pool_over_samples(feats: torch.Tensor, pooling: str, grouped_xyz=None, sigma=None, nsample=None):
    """(B, C, npoint, nsample) -> (B, C, npoint)."""
    if pooling == "max":
        return F.max_pool2d(feats, kernel_size=[1, feats.size(3)]).squeeze(-1)
    if pooling == "avg":
        return F.avg_pool2d(feats, kernel_size=[1, feats.size(3)]).squeeze(-1)
    if pooling == "rbf":
        # reference pointnet2_modules.py:258-262
        rbf = torch.exp(-1 * grouped_xyz.pow(2).sum(1, keepdim=False) / (sigma ** 2) / 2)
        return torch.sum(feats * rbf.unsqueeze(1), -1) / float(nsample)
    raise ValueError(f"unknown pooling {pooling}")


class _PointnetSAModuleBase(nn.Module):
    def __init__(self):
        super().__init__()
        self.npoint = None
        self.groupers = None
        self.mlps = None

    def forward(self, xyz: torch.Tensor, features: Optional[torch.Tensor] = None):
        """xyz (B, N, 3), features (B, C, N) -> new_xyz (B, npoint, 3), new_features (B, sum C_out, npoint)."""
        xyz_flipped = xyz.transpose(1, 2).contiguous()
        new_xyz = None
        if self.npoint is not None:
            inds = pointnet2_utils.furthest_point_sample(xyz, self.npoint)
            new_xyz = pointnet2_utils.gather_operation(xyz_flipped, inds).transpose(1, 2).contiguous()
        outs = []
        for grouper, mlp in zip(self.groupers, self.mlps):
            outs.append(_pool_over_samples(mlp(grouper(xyz, new_xyz, features)), "max"))
        return new_xyz, torch.cat(outs, dim=1)


class PointnetSAModuleMSG(_PointnetSAModuleBase):
    """Multi-scale grouping SA layer (reference pointnet2_modules.py:72-129)."""

    def __init__(self, *, npoint: int, radii: List[float], nsamples: List[int], mlps: List[List[int]],
                 bn: bool = True, use_xyz: bool = True, sample_uniformly: bool = False):
        super().__init__()
        assert len(radii) == len(nsamples) == len(mlps)
        self.npoint = npoint
        self.groupers = nn.ModuleList()
        self.mlps = nn.ModuleList()
        for radius, nsample, spec in zip(radii, nsamples, mlps):
            self.groupers.append(
                pointnet2_utils.QueryAndGroup(radius, nsample, use_xyz=use_xyz, sample_uniformly=sample_uniformly)
                if npoint is not None else pointnet2_utils.GroupAll(use_xyz))
            if use_xyz:
                spec[0] += 3  # the reference mutates the caller's list too
            self.mlps.append(pt_utils.SharedMLP(spec, bn=bn))


class PointnetSAModule(PointnetSAModuleMSG):
    """Single-scale SA layer (reference pointnet2_modules.py:132-163)."""

    def __init__(self, *, mlp: List[int], npoint: int = None, radius: float = None, nsample: int = None,
                 bn: bool = True, use_xyz: bool = True):
        super().__init__(mlps=[mlp], npoint=npoint, radii=[radius], nsamples=[nsample], bn=bn, use_xyz=use_xyz)


class PointnetSAModuleVotes(nn.Module):
    """SA layer that also returns the sampled indices -- the 3DETR pre-encoder.

    Contract of reference pointnet2_modules.py:161-268:
        forward(xyz (B, N, 3), features (B, C, N) | None, inds (B, npoint) | None)
            -> new_xyz (B, npoint, 3), new_features (B, mlp[-1], npoint), inds (B, npoint) [, unique_cnt]
    Hot path on the H100: cluster FPS kernel -> gather -> fused ball-query/group/
    normalise kernel -> shared MLP -> max over the ball.
    """

    def __init__(self, *, mlp: List[int], npoint: int = None, radius: float = None, nsample: int = None,
                 bn: bool = True, use_xyz: bool = True, pooling: str = "max", sigma: float = None,
                 normalize_xyz: bool = False, sample_uniformly: bool = False, ret_unique_cnt: bool = False):
        super().__init__()
        self.npoint = npoint
        self.radius = radius
        self.nsample = nsample
        self.pooling = pooling
        self.mlp_module = None
        self.use_xyz = use_xyz
        self.sigma = sigma if sigma is not None else (self.radius / 2 if self.radius is not None else None)
        self.normalize_xyz = normalize_xyz
        self.ret_unique_cnt = ret_unique_cnt

        if npoint is not None:
            self.grouper = pointnet2_utils.QueryAndGroup(
                radius, nsample, use_xyz=use_xyz, ret_grouped_xyz=True, normalize_xyz=normalize_xyz,
                sample_uniformly=sample_uniformly, ret_unique_cnt=ret_unique_cnt)
        else:
            self.grouper = pointnet2_utils.GroupAll(use_xyz, ret_grouped_xyz=True)

        mlp_spec = mlp
        if use_xyz and len(mlp_spec) > 0:
            mlp_spec[0] += 3  # in place, as the reference does (pointnet2_modules.py:200-202)
        self.mlp_module = pt_utils.SharedMLP(mlp_spec, bn=bn)

    def forward(self, xyz: torch.Tensor, features: Optional[torch.Tensor] = None,
                inds: Optional[torch.Tensor] = None):
        xyz_flipped = xyz.transpose(1, 2).contiguous()
        if inds is None:
            inds = pointnet2_utils.furthest_point_sample(xyz, self.npoint)
        else:
            assert inds.shape[1] == self.npoint
        new_xyz = None
        if self.npoint is not None:
            new_xyz = pointnet2_utils.gather_operation(xyz_flipped, inds).transpose(1, 2).contiguous()

        unique_cnt = None
        if not self.ret_unique_cnt:
            grouped_features, grouped_xyz = self.grouper(xyz, new_xyz, features)
        else:
            grouped_features, grouped_xyz, unique_cnt = self.grouper(xyz, new_xyz, features)

        new_features = self.mlp_module.forward_max_pooled(grouped_features) if self.pooling == "max" else None
        if new_features is None and self.pooling == "max":
            new_features = self.mlp_module.forward_max_pooled_infer(grouped_features)   # eval mode, no autograd
        if new_features is None:
            new_features = self.mlp_module(grouped_features)  # (B, mlp[-1], npoint, nsample)
            new_features = _pool_over_samples(new_features, self.pooling, grouped_xyz, self.sigma, self.nsample)

        if not self.ret_unique_cnt:
            return new_xyz, new_features, inds
        return new_xyz, new_features, inds, unique_cnt


class PointnetSAModuleMSGVotes(nn.Module):
    """Multi-scale variant returning indices (reference pointnet2_modules.py:270-349)."""

    def __init__(self, *, mlps: List[List[int]], npoint: int, radii: List[float], nsamples: List[int],
                 bn: bool = True, use_xyz: bool = True, sample_uniformly: bool = False):
        super().__init__()
        assert len(mlps) == len(nsamples) == len(radii)
        self.npoint = npoint
        self.groupers = nn.ModuleList()
        self.mlps = nn.ModuleList()
        for radius, nsample, spec in zip(radii, nsamples, mlps):
            self.groupers.append(
                pointnet2_utils.QueryAndGroup(radius, nsample, use_xyz=use_xyz, sample_uniformly=sample_uniformly)
                if npoint is not None else pointnet2_utils.GroupAll(use_xyz))
            if use_xyz:
                spec[0] += 3
            self.mlps.append(pt_utils.SharedMLP(spec, bn=bn))

    def forward(self, xyz: torch.Tensor, features: Optional[torch.Tensor] = None,
                inds: Optional[torch.Tensor] = None):
        xyz_flipped = xyz.transpose(1, 2).contiguous()
        if inds is None:
            inds = pointnet2_utils.furthest_point_sample(xyz, self.npoint)
        new_xyz = None
        if self.npoint is not None:
            new_xyz = pointnet2_utils.gather_operation(xyz_flipped, inds).transpose(1, 2).contiguous()
        outs = [_pool_over_samples(mlp(grouper(xyz, new_xyz, features)), "max")
                for grouper, mlp in zip(self.groupers, self.mlps)]
        return new_xyz, torch.cat(outs, dim=1), inds


class PointnetFPModule(nn.Module):
    """Feature propagation by inverse-distance three-NN interpolation
    (reference pointnet2_modules.py:352-412)."""

    def __init__(self, *, mlp: List[int], bn: bool = True):
        super().__init__()
        self.mlp = pt_utils.SharedMLP(mlp, bn=bn)

    def forward(self, unknown: torch.Tensor, known: torch.Tensor, unknow_feats: torch.Tensor,
                known_feats: torch.Tensor) -> torch.Tensor:
        if known is not None:
            dist, idx = pointnet2_utils.three_nn(unknown, known)
            dist_recip = 1.0 / (dist + 1e-8)
            weight = dist_recip / torch.sum(dist_recip, dim=2, keepdim=True)
            interpolated = pointnet2_utils.three_interpolate(known_feats, idx, weight)
        else:
            interpolated = known_feats.expand(*known_feats.size()[0:2], unknown.size(1))
        new_features = interpolated if unknow_feats is None else torch.cat([interpolated, unknow_feats], dim=1)
        return self.mlp(new_features.unsqueeze(-1)).squeeze(-1)


class PointnetLFPModuleMSG(nn.Module):
    """Learnable feature propagation with multi-scale grouping
    (reference pointnet2_modules.py:414-492)."""

    def __init__(self, *, mlps: List[List[int]], radii: List[float], nsamples: List[int],
                 post_mlp: List[int], bn: bool = True, use_xyz: bool = True, sample_uniformly: bool = False):
        super().__init__()
        assert len(mlps) == len(nsamples) == len(radii)
        self.post_mlp = pt_utils.SharedMLP(post_mlp, bn=bn)
        self.groupers = nn.ModuleList()
        self.mlps = nn.ModuleList()
        for radius, nsample, spec in zip(radii, nsamples, mlps):
            self.groupers.append(pointnet2_utils.QueryAndGroup(radius, nsample, use_xyz=use_xyz,
                                                               sample_uniformly=sample_uniformly))
            if use_xyz:
                spec[0] += 3
            self.mlps.append(pt_utils.SharedMLP(spec, bn=bn))

    def forward(self, xyz2: torch.Tensor, xyz1: torch.Tensor, features2: torch.Tensor,
                features1: torch.Tensor) -> torch.Tensor:
        outs = []
        for grouper, mlp in zip(self.groupers, self.mlps):
            f = grouper(xyz1, xyz2, features1)
            f = _pool_over_samples(mlp(f), "max")
            if features2 is not None:
                f = torch.cat([f, features2], dim=1)
            outs.append(self.post_mlp(f.unsqueeze(-1)))
        return torch.cat(outs, dim=1).squeeze(-1)
