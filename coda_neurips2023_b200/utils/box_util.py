"""Box geometry on the hot path (reference utils/box_util.py).

Corner builders are the same closed forms as the reference's
`get_3d_box_batch_tensor` (:440-490) / `get_3d_box_batch_tensor_xyz` (:383-423)
written without the scatter-into-zeros idiom; GIoU runs in one CUDA kernel
(ops.giou3d) instead of tensor code + Cython on the host.
"""
from __future__ import annotations

import torch

from .. import ops

# sign pattern of the 8 corners: reference box_util.py:466-474 (camera frame) and :409-417 (upright xyz)
_SX_CAM = (1, 1, -1, -1, 1, 1, -1, -1)
_SY_CAM = (1, 1, 1, 1, -1, -1, -1, -1)
_SZ_CAM = (1, -1, -1, 1, 1, -1, -1, 1)
_SX_XYZ = (-1, 1, 1, -1, -1, 1, 1, -1)
_SY_XYZ = (1, 1, -1, -1, 1, 1, -1, -1)
_SZ_XYZ = (1, 1, 1, 1, -1, -1, -1, -1)


def flip_axis_to_camera_tensor(pc: torch.Tensor) -> torch.Tensor:
    """depth (X right, Y forward, Z up) -> camera (X right, Y down, Z forward)."""
    return torch.stack((pc[..., 0], -pc[..., 2], pc[..., 1]), dim=-1)


_SIGN_CACHE: dict = {}


def _signs(t, like):
    """Corner sign pattern as a tensor on `like`'s device, built once per (pattern, device, dtype):
    a host->device copy per call would also be illegal inside a CUDA-graph capture."""
    key = (t, like.device, like.dtype)
    if key not in _SIGN_CACHE:
        _SIGN_CACHE[key] = torch.tensor(t, dtype=like.dtype, device=like.device)
    return _SIGN_CACHE[key]


def get_3d_box_batch_tensor(box_size, angle, center):
    """Corners in the camera frame: box_size (..., 3) = (l, w, h), heading `angle`
    about camera Y, `center` (..., 3) already flipped to the camera frame -> (..., 8, 3)."""
    l, w, h = box_size[..., 0:1] / 2, box_size[..., 1:2] / 2, box_size[..., 2:3] / 2
    x = l * _signs(_SX_CAM, box_size)
    y = h * _signs(_SY_CAM, box_size)
    z = w * _signs(_SZ_CAM, box_size)
    c, s = torch.cos(angle)[..., None], torch.sin(angle)[..., None]
    # corners @ roty(angle)^T with roty = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
    out = torch.stack((x * c + z * s, y, -x * s + z * c), dim=-1)
    return out + center[..., None, :]


def get_3d_box_batch_tensor_xyz(box_size, angle, center):
    """Corners in the upright depth frame (rotation about Z by -angle) -> (..., 8, 3)."""
    l, w, h = box_size[..., 0:1] / 2, box_size[..., 1:2] / 2, box_size[..., 2:3] / 2
    x = l * _signs(_SX_XYZ, box_size)
    y = w * _signs(_SY_XYZ, box_size)
    z = h * _signs(_SZ_XYZ, box_size)
    c, s = torch.cos(-angle)[..., None], torch.sin(-angle)[..., None]
    # corners @ rotz(-angle)^T with rotz = [[c, -s, 0], [s, c, 0], [0, 0, 1]]
    out = torch.stack((x * c - y * s, x * s + y * c, z), dim=-1)
    return out + center[..., None, :]


def generalized_box3d_iou(corners1, corners2, nums_k2, rotated_boxes: bool = True,
                          return_inter_vols_only: bool = False, needs_grad: bool = False,
                          rot_k2_limit=None):
    """(B, K1, 8, 3), (B, K2, 8, 3), (B,) -> GIoU (B, K1, K2), no grad.

    `rot_k2_limit=4` reproduces the compiled-Cython reference, which clips rotated
    rectangles only for gt index < 4 (utils/box_intersection.pyx:181); the default
    computes every pair like the reference's TorchScript path."""
    if needs_grad or return_inter_vols_only:
        raise NotImplementedError("differentiable GIoU (loss_giou_weight > 0) is not on the device path; "
                                  "every shipped CoDA script sets loss_giou_weight 0")
    rot = rotated_boxes if isinstance(rotated_boxes, torch.Tensor) else bool(rotated_boxes)
    return ops.giou3d(corners1.detach(), corners2.detach(), nums_k2, rot, rot_k2_limit)
