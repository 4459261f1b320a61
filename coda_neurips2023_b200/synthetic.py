"""Seeded synthetic SUN RGB-D / ScanNet-shaped inputs (SURVEY.md section 8d).

There is no dataset offline; every test and the benchmark draw their scenes
from here.  Shapes and dtypes follow what the reference's dataloader collates
(datasets/sunrgbd_anonymous_aligned_image.py:813-899).
"""
from __future__ import annotations

import numpy as np

ROOM_MIN = np.array([-3.0, 0.5, -1.2], dtype=np.float32)
ROOM_MAX = np.array([3.0, 6.0, 1.5], dtype=np.float32)


def point_clouds(batch: int, npoints: int, seed: int = 0, dup_frac: float = 0.01,
                 near_origin: int = 3) -> np.ndarray:
    """(batch, npoints, 3) fp32 points uniform in a 6 x 5.5 x 2.7 m room, with
    `dup_frac` exact duplicates (the reference resamples WITH replacement when a
    scan has fewer than 20 000 points, utils/pc_util.py:24-32) and a few points
    with |p|^2 <= 1e-3, which FPS must skip (sampling_gpu.cu:104)."""
    rng = np.random.default_rng(seed)
    pc = rng.uniform(ROOM_MIN, ROOM_MAX, size=(batch, npoints, 3)).astype(np.float32)
    ndup = int(npoints * dup_frac)
    for b in range(batch):
        if ndup > 0 and npoints > 1:
            dst = rng.choice(npoints, size=ndup, replace=False)
            src = rng.integers(0, npoints, size=ndup)
            pc[b, dst] = pc[b, src]
        k = min(near_origin, max(npoints - 1, 0))
        if k > 0:
            where = rng.choice(np.arange(1, npoints), size=k, replace=False)
            pc[b, where] = rng.uniform(-0.015, 0.015, size=(k, 3)).astype(np.float32)
    return pc


# ---------------------------------------------------------------------------
#  Synthetic training batches, argument namespace and dataset config
# ---------------------------------------------------------------------------
import argparse  # noqa: E402


class SyntheticDatasetConfig:
    """The attributes / methods of the reference's dataset config objects that the model
    and the criterion touch (datasets/sunrgbd_anonymous_aligned_image.py:86-300)."""

    def __init__(self, args=None, num_semcls: int = 1, num_angle_bin: int = 12, max_num_obj: int = 64):
        self.num_semcls = num_semcls
        self.num_angle_bin = num_angle_bin
        self.max_num_obj = max_num_obj
        self.image_size = [getattr(args, "image_size_width", 730), getattr(args, "image_size_height", 531)]

    def box_parametrization_to_corners(self, box_center_unnorm, box_size, box_angle):
        from .utils.box_util import flip_axis_to_camera_tensor, get_3d_box_batch_tensor

        return get_3d_box_batch_tensor(box_size, box_angle, flip_axis_to_camera_tensor(box_center_unnorm))

    def box_parametrization_to_corners_xyz(self, box_center_unnorm, box_size, box_angle):
        from .utils.box_util import get_3d_box_batch_tensor_xyz

        return get_3d_box_batch_tensor_xyz(box_size, box_angle, box_center_unnorm)


SCANNET_TRAIN_RANGE_LIST = (2, 4, 5, 7, 13, 15, 16, 22, 56, 1163)
SCANNET_TEST_RANGE_LIST = (
    2, 4, 5, 6, 7, 8, 9, 10, 11, 13, 14, 15, 16, 17, 18, 19, 21, 22, 23, 24, 26, 27, 28, 29, 31, 32, 33, 34, 35, 36,
    38, 39, 40, 41, 42, 44, 45, 46, 47, 48, 49, 50, 51, 52, 54, 55, 56, 57, 58, 59, 62, 63, 64, 65, 66, 67, 68, 69,
    70, 71, 72, 73, 74, 75, 76, 77, 78, 79, 80, 82, 84, 86, 87, 88, 89, 90, 93, 95, 96, 97, 98, 99, 100, 101, 102,
    103, 104, 105, 106, 107, 110, 112, 115, 116, 118, 120, 121, 122, 125, 128, 130, 131, 132, 134, 136, 138, 139,
    140, 141, 145, 148, 154, 155, 156, 157, 159, 161, 163, 165, 166, 168, 169, 170, 177, 180, 185, 188, 191, 193,
    195, 202, 208, 213, 214, 221, 229, 230, 232, 233, 242, 250, 261, 264, 276, 283, 286, 300, 304, 312, 323, 325,
    331, 342, 356, 370, 392, 395, 399, 408, 417, 488, 540, 562, 570, 572, 581, 609, 748, 776, 1156, 1163, 1164,
    1165, 1166, 1167, 1168, 1169, 1170, 1171, 1172, 1173, 1174, 1175, 1176, 1178, 1179, 1180, 1181, 1182, 1183,
    1184, 1185, 1186, 1187, 1188, 1189, 1190, 1191)


def make_args(**overrides) -> argparse.Namespace:
    """Defaults of the reference's main.py argument parser (main.py:37-304) for every field
    the model / criterion read, overlaid with scripts/coda_sunrgbd_stage1.sh, overlaid with
    `overrides`.  nqueries defaults to the BASELINE metric's 256."""
    a = dict(
        # model (main.py:69-74, :127-143; stage1 script)
        model_name="3detr_predictedbox_distillation", dataset_name="sunrgbd_anonymous_aligned_image",
        enc_type="vanilla", enc_nlayers=3, enc_dim=256, enc_ffn_dim=128, enc_dropout=0.1, enc_nhead=4,
        enc_activation="relu", dec_nlayers=8, dec_dim=512, dec_ffn_dim=256, dec_dropout=0.1, dec_nhead=4,
        mlp_dropout=0.3, nqueries=256, preenc_npoints=2048, use_color=False,
        if_use_v1=True, if_clip_more_prompts=True, if_clip_superset=False, if_clip_weak_labels=False,
        train_range_max=10, test_range_max=46, distillation_box_num=32, keep_objectness=0.5,
        image_size_width=730, image_size_height=531, clip_arch="ViT-B/32",
        clip_checkpoint="./CLIP/pretrain_models/ViT-B-16.pt",
        # matcher / losses (stage1 script)
        matcher_giou_cost=3.0, matcher_cls_cost=1.0, matcher_center_cost=5.0, matcher_objectness_cost=5.0,
        loss_giou_weight=0.0, loss_sem_cls_weight=0.0, loss_sem_cls_softmax_weight=0.0,
        loss_sem_cls_softmax_skip_none_gt_sample_weight=1.0, loss_no_object_weight=0.05,
        loss_angle_cls_weight=0.1, loss_angle_reg_weight=0.5, loss_center_weight=5.0, loss_size_weight=1.0,
        loss_no_object_contrast_weight=0.05, loss_predicted_region_embed_l1_weight=1.0,
        confidence_type="non-confidence",
        # optimiser (main.py:41-52; stage1 script)
        base_lr=1.97e-4, warm_lr=1e-6, warm_lr_epochs=18, final_lr=1e-6, lr_scheduler="cosine",
        weight_decay=0.1, filter_biases_wd=False, clip_gradient=0.1, max_epoch=1080,
        batchsize_per_gpu=8, ngpus=1,
        # ScanNet-200 class ids of the seen / evaluated prompts and the cap on added unseen classes (main.py:245-247;
        # scripts/coda_scannet_stage1.sh); read only when dataset_name names ScanNet
        train_range_list=list(SCANNET_TRAIN_RANGE_LIST), test_range_list=list(SCANNET_TEST_RANGE_LIST),
        reset_scannet_num=50,
    )
    a.update(overrides)
    return argparse.Namespace(**a)


def _corners_np(size, angle, center_cam):
    """(..., 8, 3) camera-frame corners in numpy (same closed form as utils/box_util.py)."""
    sx = np.array((1, 1, -1, -1, 1, 1, -1, -1), np.float32)
    sy = np.array((1, 1, 1, 1, -1, -1, -1, -1), np.float32)
    sz = np.array((1, -1, -1, 1, 1, -1, -1, 1), np.float32)
    x = size[..., 0:1] / 2 * sx
    y = size[..., 2:3] / 2 * sy
    z = size[..., 1:2] / 2 * sz
    c, s = np.cos(angle)[..., None], np.sin(angle)[..., None]
    out = np.stack((x * c + z * s, y, -x * s + z * c), -1)
    return (out + center_cam[..., None, :]).astype(np.float32)


def make_batch(batch: int, npoints: int = 20000, seed: int = 0, max_gt: int = 64, image_hw=(531, 730),
               num_angle_bin: int = 12, ncls_seen: int = 10, min_gt: int = 3, max_real_gt: int = 20,
               camera: str = "sunrgbd"):
    """One SUN RGB-D-shaped training batch as numpy arrays / what the dataloader collates
    (datasets/sunrgbd_anonymous_aligned_image.py:813-899; SURVEY.md section 8d).  fp64 where
    the reference's numpy arrays are fp64 (K, Rtilt, rot_array, scale_array, flip arrays).
    camera="scannet": the image side of a ScanNet batch instead (datasets/scannet_anonymous_aligned_image.py:537-702,
    see _scannet_camera); the point cloud and the boxes are drawn the same way."""
    if camera not in ("sunrgbd", "scannet"):
        raise ValueError(f"unknown camera {camera!r}")
    rng = np.random.default_rng(seed + 7919)
    pc = point_clouds(batch, npoints, seed=seed)
    h, w = image_hw
    d = {
        "point_clouds": pc,
        "point_cloud_dims_min": pc.min(axis=1),
        "point_cloud_dims_max": pc.max(axis=1),
    }
    present = np.zeros((batch, max_gt), np.float32)
    centers = np.zeros((batch, max_gt, 3), np.float32)
    sizes = np.zeros((batch, max_gt, 3), np.float32)
    angles = np.zeros((batch, max_gt), np.float32)
    for b in range(batch):
        n = int(rng.integers(min_gt, max_real_gt + 1))
        present[b, :n] = 1
        centers[b, :n] = rng.uniform(ROOM_MIN + 0.3, ROOM_MAX - 0.3, size=(n, 3))
        sizes[b, :n] = rng.uniform(0.3, 2.0, size=(n, 3))
        angles[b, :n] = rng.uniform(-np.pi, np.pi, size=n)
    per_cls = 2 * np.pi / num_angle_bin
    shifted = (angles % (2 * np.pi) + per_cls / 2) % (2 * np.pi)
    cls = (shifted / per_cls).astype(np.int64)
    res = (shifted - (cls * per_cls + per_cls / 2)).astype(np.float32)
    span = d["point_cloud_dims_max"] - d["point_cloud_dims_min"]
    cam = np.stack((centers[..., 0], -centers[..., 2], centers[..., 1]), -1)
    d.update({
        "gt_box_present": present,
        "gt_box_centers": centers,
        "gt_box_centers_normalized": ((centers - d["point_cloud_dims_min"][:, None]) / span[:, None]).astype(np.float32),
        "gt_box_sizes": sizes,
        "gt_box_sizes_normalized": (sizes / np.clip(span, 0.1, None)[:, None]).astype(np.float32),
        "gt_box_angles": angles * present,
        "gt_angle_class_label": cls * present.astype(np.int64),
        "gt_angle_residual_label": res * present,
        "gt_box_corners": _corners_np(sizes, angles, cam) * present[..., None, None],
        "gt_box_sem_cls_label": np.zeros((batch, max_gt), np.int64),
        "gt_box_seen_sem_cls_label": rng.integers(0, ncls_seen, size=(batch, max_gt)).astype(np.int64),
        "gt_box_seen_sem_cls_confi": present.copy(),
    })
    if camera == "scannet":
        d.update(_scannet_camera(rng, batch, h, w))
        d["gt_ori_box_num"] = present.sum(axis=1).astype(np.int64)
        return d
    # image side: SUN RGB-D-like intrinsics, small tilt, augmentation bookkeeping
    # SUN RGB-D intrinsics at 730 x 531; other image shapes (ScanNet: 1296 x 968) scale the focal length with
    # the width and keep the principal point at the same relative position
    f = 529.5 * w / 730.0
    K = np.tile(np.array([[f, 0, 365.0 * w / 730.0], [0, f, 265.0 * h / 531.0], [0, 0, 1.0]]), (batch, 1, 1))
    tilt = rng.uniform(-0.05, 0.05, size=batch)
    Rtilt = np.stack([np.array([[1, 0, 0], [0, np.cos(t), -np.sin(t)], [0, np.sin(t), np.cos(t)]]) for t in tilt])
    rot = rng.uniform(-np.pi / 18, np.pi / 18, size=batch)
    rot_array = np.stack([np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1.0]]) for t in rot])
    d.update({
        "input_image": rng.integers(0, 256, size=(batch, h, w, 3), dtype=np.uint8),
        "K": K.astype(np.float64), "Rtilt": Rtilt.astype(np.float64), "rot_array": rot_array.astype(np.float64),
        "flip_array": rng.choice([-1.0, 1.0], size=(batch, 1)).astype(np.float64),
        "scale_array": rng.uniform(0.9, 1.1, size=(batch, 1, 1)).repeat(3, axis=2).astype(np.float64),
        "image_flip_array": rng.choice([0.0, 1.0], size=(batch, 1)).astype(np.float64),
        "flip_length": np.full((batch,), float(w), np.float64),
        "ori_width": np.full((batch,), w, np.int64), "ori_height": np.full((batch,), h, np.int64),
        "x_offset": np.zeros((batch,), np.int64), "y_offset": np.zeros((batch,), np.int64),
        # stage 2 (novel-box discovery) reads these as well (model_3detr.py:1228, :1515)
        "rot_angle": rot.astype(np.float64),
        "gt_ori_box_num": present.sum(axis=1).astype(np.int64),
    })
    return d


def rotz(t: float) -> np.ndarray:
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


# ScanNet colour-camera intrinsics (intrinsic/intrinsic_color.txt of a typical scene, 1296 x 968)
SCANNET_COLOR_FOCAL = 1170.19
SCANNET_COLOR_CENTER = (647.75, 483.75)
SCANNET_CAMERA_DISTANCE = (-1.2, -0.8)     # along the heading of the room's centre from the origin, m


def _scannet_camera(rng, batch: int, h: int, w: int) -> dict:
    """Image side of a ScanNet batch (datasets/scannet_anonymous_aligned_image.py:537-702): K the 4 x 4 colour
    intrinsics scaled to the image size, Rtilt the 4 x 4 camera-to-world pose, and ScanNet's augmentation
    bookkeeping (x flip, zx flip, rotation within +-30 degrees with rot_array = inv(rotz^T), scale).

    The pose lives in the scene's frame before augmentation, where the flips and the rotation put the synthetic
    room anywhere around the origin.  The camera stands 1.5 m above the room's floor, 0.8 .. 1.2 m behind the origin
    as seen from the room's centre, and looks towards the centre with a small yaw and a downward pitch; the camera
    frame is x right, y down, z forward, as in ScanNet.  With the metre-sized boxes of an untrained model this
    gives, in every scene, boxes inside the image, boxes clipped at an image edge and boxes behind the camera."""
    rot = rng.uniform(-np.pi / 6, np.pi / 6, size=batch)
    rot_array = np.stack([np.linalg.inv(rotz(t).T) for t in rot])
    flip = rng.choice([-1.0, 1.0], size=(batch, 1)).astype(np.float64)
    zx_flip = rng.choice([-1.0, 1.0], size=(batch, 1)).astype(np.float64)
    scale = rng.uniform(0.9, 1.1, size=(batch, 1, 1)).repeat(3, axis=2).astype(np.float64)
    image_flip = rng.choice([0.0, 1.0], size=(batch, 1)).astype(np.float64)
    yaw = rng.uniform(-np.pi / 12, np.pi / 12, size=batch)
    pitch = rng.uniform(np.pi / 36, np.pi / 9, size=batch)               # 5 .. 20 degrees down
    dist = rng.uniform(*SCANNET_CAMERA_DISTANCE, size=batch)
    height = rng.uniform(-0.1, 0.1, size=batch)
    sx, sy = w / 1296.0, h / 968.0
    K = np.zeros((batch, 4, 4))
    K[:, 0, 0], K[:, 1, 1] = SCANNET_COLOR_FOCAL * sx, SCANNET_COLOR_FOCAL * sy
    K[:, 0, 2], K[:, 1, 2] = SCANNET_COLOR_CENTER[0] * sx, SCANNET_COLOR_CENTER[1] * sy
    K[:, 2, 2] = K[:, 3, 3] = 1.0
    pose = np.zeros((batch, 4, 4))
    for b in range(batch):
        centre = (0.5 * (ROOM_MIN + ROOM_MAX)).astype(np.float64) * scale[b, 0] @ rot_array[b]   # augmentation undone
        centre[1] *= zx_flip[b, 0]
        centre[0] *= flip[b, 0]
        head = np.arctan2(centre[0], centre[1])                           # heading of the centre, from +y towards +x
        fwd = np.array([np.sin(head + yaw[b]) * np.cos(pitch[b]), np.cos(head + yaw[b]) * np.cos(pitch[b]),
                        -np.sin(pitch[b])])
        right = np.array([np.cos(head + yaw[b]), -np.sin(head + yaw[b]), 0.0])
        pose[b, :3, :3] = np.stack((right, np.cross(fwd, right), fwd), axis=1)   # columns: camera axes in the world
        pose[b, :3, 3] = (dist[b] * np.sin(head), dist[b] * np.cos(head), ROOM_MIN[2] + 1.5 + height[b])
        pose[b, 3, 3] = 1.0
    # a pose read from text is not exactly orthonormal: keep it as printed with 6 decimals
    pose = np.round(pose, 6)
    return {
        "input_image": rng.integers(0, 256, size=(batch, h, w, 3), dtype=np.uint8),
        "K": K, "Rtilt": pose, "rot_array": rot_array, "flip_array": flip, "zx_flip_array": zx_flip,
        "scale_array": scale, "image_flip_array": image_flip,
        "flip_length": np.full((batch,), float(w), np.float64),
        "ori_width": np.full((batch,), w, np.int64), "ori_height": np.full((batch,), h, np.int64),
        "x_offset": np.zeros((batch,), np.int64), "y_offset": np.zeros((batch,), np.int64),
        "rot_angle": rot.astype(np.float64),
    }


def to_device(batch_np: dict, device, pinned: bool = False) -> dict:
    """What engine.py:125-129 does with a collated batch: every array -> tensor on `device`."""
    import torch

    out = {}
    for k, v in batch_np.items():
        t = torch.from_numpy(np.ascontiguousarray(v))
        if pinned:
            t = t.pin_memory()
        out[k] = t.to(device, non_blocking=pinned)
    return out
