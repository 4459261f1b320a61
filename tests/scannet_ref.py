"""The reference's ScanNet crop projection as its own chain of fp64 tensor ops, for the CPU tests and the GPU checks of
ops.boxes_in_image(camera="scannet").  TEST INFRASTRUCTURE ONLY, like oracle/cpu_step.py, whose SUN RGB-D
restatement (`cpu_step._boxes_in_image`) it dispatches to for the SUN RGB-D camera.

ScanNet (reference datasets/scannet_utils.py:650-690, called from models/model_3detr.py:931 and :1255): K is the 4x4
colour intrinsics, Rtilt the 4x4 camera-to-world pose; p_cam = inv(pose) [p, 1] (torch.linalg.inv, fp64, no axis
swap), uv = K[:3, :3] p_cam, pixel = uv[0:2] / (uv[2] + 1e-32), depth = uv[2].  The steps before (undo scale,
rot_array, zx flip, x flip; :912-930) and after (clip to the original image, offsets, image flip; :950-968) are the
same as for SUN RGB-D."""
from __future__ import annotations

import contextlib

import torch

import cpu_step


def undo_point_augmentation(corners_xyz, inputs):
    """Scale, rot_array, the zx flip and the x flip undone (models/model_3detr.py:912-930), fp64 (B, Q, 8, 3)."""
    pts = corners_xyz.to(torch.double) * inputs["scale_array"].unsqueeze(1).to(torch.double)
    pts = torch.matmul(pts, inputs["rot_array"].unsqueeze(1).to(torch.double))
    if "zx_flip_array" in inputs:
        pts = torch.cat((pts[..., :1], pts[..., 1:2] * inputs["zx_flip_array"].view(-1, 1, 1, 1), pts[..., 2:]), -1)
    flip = inputs["flip_array"].to(torch.double).view(-1, 1, 1, 1)
    return torch.cat((pts[..., :1] * flip, pts[..., 1:]), dim=-1)


def scannet_uv(pts, inputs):
    """project_3dpoint_to_2dpoint_corners_tensor of datasets/scannet_utils.py on fp64 points (B, Q, 8, 3) ->
    u, v (pixels before clipping), depth, each (B, Q, 8)."""
    K = inputs["K"].unsqueeze(1).to(torch.double)
    pose_inv = torch.linalg.inv(inputs["Rtilt"].unsqueeze(1).to(torch.double))
    hom = torch.cat((pts, torch.ones_like(pts[..., :1])), dim=-1)
    pc2 = torch.matmul(pose_inv, hom.transpose(2, 3)).transpose(2, 3)[..., :3]
    uv = torch.matmul(K[..., :3, :3], pc2.transpose(2, 3)).transpose(2, 3)
    depth = uv[..., 2]
    return uv[..., 0] / (depth + 1e-32), uv[..., 1] / (depth + 1e-32), depth


def project_corners_to_image(corners_xyz, inputs):
    """ScanNet camera: (B, Q, 8, 3) -> uv (B, Q, 8, 2) in the augmented image, fp64, and depth (B, Q, 8)."""
    u, v, depth = scannet_uv(undo_point_augmentation(corners_xyz, inputs), inputs)
    wmax = (inputs["ori_width"].to(torch.double) - 1).view(-1, 1, 1)
    hmax = (inputs["ori_height"].to(torch.double) - 1).view(-1, 1, 1)
    zero = torch.zeros((), dtype=torch.double, device=u.device)
    u = torch.minimum(torch.maximum(u, zero), wmax) + inputs["y_offset"].to(torch.double).view(-1, 1, 1)
    v = torch.minimum(torch.maximum(v, zero), hmax) + inputs["x_offset"].to(torch.double).view(-1, 1, 1)
    img_flip = inputs["image_flip_array"].to(torch.double).view(-1, 1, 1)
    flip_len = inputs["flip_length"].to(torch.double).view(-1, 1, 1)
    u = u * img_flip + (1 - img_flip) * (flip_len - 1 - u)
    return torch.stack((u, v), dim=-1), depth


def boxes_in_image(corners_xyz, size_unnorm, inputs, camera="sunrgbd", extent=False):
    """CPU stand-in for ops.boxes_in_image with the same signature: integer boxes (truncation), usability flags and,
    with `extent`, the fp64 [umin, vmin, umax, vmax] that are truncated."""
    if camera == "scannet":
        uv, depth = project_corners_to_image(corners_xyz, inputs)
    elif camera == "sunrgbd":
        uv, depth = cpu_step._project_corners_to_image(corners_xyz, inputs)
    else:
        raise ValueError(f"unknown camera {camera!r}")
    ext = torch.stack((uv[..., 0].amin(-1), uv[..., 1].amin(-1), uv[..., 0].amax(-1), uv[..., 1].amax(-1)), dim=-1)
    box = ext.to(torch.int32)
    xmin, ymin, xmax, ymax = box.unbind(-1)
    valid = ((xmax - xmin) > 0) & ((ymax - ymin) > 0) & (depth.amin(-1) >= 0) & ~(size_unnorm.amax(-1) < 1e-16)
    return (box, valid, ext) if extent else (box, valid)


@contextlib.contextmanager
def installed():
    """oracle/cpu_step.installed() with ops.boxes_in_image taking the camera argument (both cameras on the CPU)."""
    from coda_neurips2023_b200 import ops

    with cpu_step.installed():
        saved = ops.boxes_in_image
        ops.boxes_in_image = boxes_in_image
        try:
            yield
        finally:
            ops.boxes_in_image = saved
