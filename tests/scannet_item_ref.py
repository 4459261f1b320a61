"""TEST INFRASTRUCTURE (checker only; nothing in the package imports this).

CPU restatement, in numpy, of the ScanNet training item the device data layer builds (DeviceScanNetAugmentor in
coda_neurips2023_b200/datasets/device_pipeline.py, include/coda_data.h): datasets/scannet_anonymous_aligned_image.py
:373-702 with the train split, augmentation, image input and image augmentation on.  It crops the RAW scene
(RandomCuboid), samples it, then flips / rotates / scales the sampled rows and the boxes, as the reference does, with
the random draws taken from the same table the device takes.  It reuses the SUN RGB-D restatement's RandomCuboid,
Feistel sampler and image augmentation (oracle/data_ref.py).  tests/golden/scannet_data_ref.npz pins it to the
reference's own __getitem__ fed those draws (tests/test_scannet_data_cpu.py).
"""
from __future__ import annotations

import numpy as np

from data_ref import M32, center_index, feistel, image_augment, mix32d, random_cuboid  # noqa: F401

def sample_positions(m: int, seed: int, nsample: int) -> np.ndarray:
    """positions in a cloud of m rows that the device sampler picks (the Feistel permutation with cycle walking when
    m >= nsample, hashed draws with replacement otherwise): the reference's `choices` of random_sampling"""
    key = int(mix32d(np.uint64(seed) ^ np.uint64(0xA511E9B3)))
    i = np.arange(nsample, dtype=np.uint64)
    if m >= nsample:
        half_bits = 1
        while (1 << (2 * half_bits)) < m:
            half_bits += 1
        j = feistel(i, half_bits, key)
        while True:
            out = j >= m
            if not out.any():
                break
            j[out] = feistel(j[out], half_bits, key)
    else:
        j = mix32d((i * np.uint64(0x9E3779B1) + np.uint64(key)) & M32) % np.uint64(m)
    return j.astype(np.int64)


def image_jitter_u(seed: int, h: int, w: int) -> np.ndarray:
    """(h, w) uniforms in [0, 1) of the jitter hash of image_augment (what np.random.random((h, w)) is in the item)"""
    t = np.arange(h * w, dtype=np.uint64)
    r = mix32d((np.uint64(seed) + t * np.uint64(0x9E3779B1)) & M32)
    return ((r >> np.uint64(8)).astype(np.float64) / 16777216.0).reshape(h, w)


def pad_image(frame: np.ndarray, image_size) -> tuple:
    """frame (h, w, 3) uint8 on a white (H, W) = image_size[::-1] canvas at ((H - h) // 2, (W - w) // 2) (:385-398)"""
    W, H = image_size
    h, w = frame.shape[:2]
    xo, yo = (H - h) // 2, (W - w) // 2
    canvas = np.full((H, W, 3), 255, np.uint8)
    canvas[xo:xo + h, yo:yo + w] = frame
    return canvas, xo, yo


def _angle2class(angle, num_class=12):        # the dataset config's angle2class, on a float32 scalar
    angle = angle % (2 * np.pi)
    angle_per_class = 2 * np.pi / float(num_class)
    shifted_angle = (angle + angle_per_class / 2) % (2 * np.pi)
    class_id = int(shifted_angle / angle_per_class)
    return class_id, shifted_angle - (class_id * angle_per_class + angle_per_class / 2)


def corners_camera(centers, sizes, angles):
    """box_parametrization_to_corners_np: (g, 3) float32 each, angles (g,) float32 -> (g, 8, 3) float64"""
    c2 = centers.copy()
    c2[..., [0, 1, 2]] = c2[..., [0, 2, 1]]
    c2[..., 1] *= -1
    R = np.zeros(angles.shape + (3, 3))
    c, s = np.cos(angles), np.sin(angles)
    R[..., 0, 0], R[..., 0, 2], R[..., 1, 1], R[..., 2, 0], R[..., 2, 2] = c, s, 1, -s, c
    l, w, h = (np.expand_dims(sizes[..., k], -1) for k in range(3))
    cor = np.zeros(angles.shape + (8, 3))
    cor[..., :, 0] = np.concatenate((l / 2, l / 2, -l / 2, -l / 2, l / 2, l / 2, -l / 2, -l / 2), -1)
    cor[..., :, 1] = np.concatenate((h / 2, h / 2, h / 2, h / 2, -h / 2, -h / 2, -h / 2, -h / 2), -1)
    cor[..., :, 2] = np.concatenate((w / 2, -w / 2, -w / 2, w / 2, w / 2, -w / 2, -w / 2, w / 2), -1)
    return np.matmul(cor, np.swapaxes(R, -1, -2)) + np.expand_dims(c2, -2)


def corners_xyz(centers, sizes, angles):
    """box_parametrization_to_corners_np_xyz: get_3d_box_batch_np_xyz(size, -angle, centre) -> (g, 8, 3) float64"""
    half = sizes / 2
    t = -(-1 * angles)
    R = np.zeros(t.shape + (3, 3))
    c, s = np.cos(t), np.sin(t)
    R[..., 0, 0], R[..., 0, 1], R[..., 1, 0], R[..., 1, 1], R[..., 2, 2] = c, -s, s, c, 1
    l, w, h = (np.expand_dims(half[..., k], -1) for k in range(3))
    cor = np.zeros(t.shape + (8, 3))
    cor[..., :, 0] = np.concatenate((-l, l, l, -l, -l, l, l, -l), -1)
    cor[..., :, 1] = np.concatenate((w, w, -w, -w, w, w, -w, -w), -1)
    cor[..., :, 2] = np.concatenate((h, h, h, h, -h, -h, -h, -h), -1)
    return np.matmul(cor, np.swapaxes(R, -1, -2)) + np.expand_dims(centers, -2)


def scannet_item(raw, bbox, frame, draws, b, select_range, image_size, num_points=40000, min_points=30000,
                 max_num_obj=64, aspect=0.8):
    """The ScanNet training item of scene b of `draws` (device_pipeline.draw_augmentation_scannet):
    raw (n, 6) float32 `_pc.npy` rows [x, y, z, r, g, b]; bbox (g, 8) float32 `_bbox.npy` rows
    [cx, cy, cz, dx/2, dy/2, dz/2, heading, class id]; frame (h, w, 3) uint8 RGB; image_size (W, H).
    -> the reference's ret_dict fields plus `chosen` (RandomCuboid attempt or -1), `box_keep` (kept rows of the
    class-filtered boxes), `list_pos` (sampled positions in the cropped cloud), `choice` (their raw rows) and
    `count` (rows in the cropped cloud)."""
    d = {k: np.asarray(v)[b] for k, v in draws.items()}
    # image (:385-398, :458-491): pad, then the image augmentation of the whole canvas
    canvas, xo, yo = pad_image(frame, image_size)
    img = image_augment(canvas, bool(d["image_flip"]), d["image_gain"], d["image_shift"], int(d["image_seed"]))
    # boxes of the selected classes, class column zeroed (:433-438)
    boxes = bbox[np.isin(bbox[:, -1], select_range)].astype(np.float32)
    boxes[:, -1] = 0
    if len(boxes) > max_num_obj:
        raise ValueError(f"{len(boxes)} boxes after the class filter; max_num_obj is {max_num_obj}")
    xyz = raw[:, 0:3]
    chosen, crop, keep = random_cuboid(xyz, boxes, d["crop_range"], d["center_u"], min_points, aspect)
    if chosen >= 0:
        rows = np.nonzero(np.all(xyz.astype(np.float64) <= crop[3:], axis=1)
                          & np.all(xyz.astype(np.float64) >= crop[:3], axis=1))[0]
    else:
        rows = np.arange(len(xyz))
    j = sample_positions(len(rows), int(d["seed"]), num_points)
    choice = rows[j]
    point_cloud = xyz[choice].copy()
    point_cloud_rgb = raw[:, 0:6][j]                                       # the uncropped scene at the crop's choices
    pcl_color = raw[:, 3:6][j]
    kept = boxes[keep]
    k = len(kept)
    target_bboxes = np.zeros((max_num_obj, 7), np.float32)
    mask = np.zeros(max_num_obj, np.float32)
    mask[:k] = 1
    target_bboxes[:k] = kept[:, 0:7]
    # flips, rotation, scale (:538-606), the reference's own statements and operand types
    flip_array, zx_flip_array = np.ones(1), np.ones(1)
    if d["flip_yz"] < 0:
        point_cloud[:, 0] = -1 * point_cloud[:, 0]
        point_cloud_rgb[:, 0] = -1 * point_cloud_rgb[:, 0]
        target_bboxes[:, 0] = -1 * target_bboxes[:, 0]
        flip_array = flip_array * -1
        target_bboxes[:, 6] = np.pi - target_bboxes[:, 6]
    if d["flip_xz"] < 0:
        point_cloud[:, 1] = -1 * point_cloud[:, 1]
        point_cloud_rgb[:, 1] = -1 * point_cloud_rgb[:, 1]
        target_bboxes[:, 1] = -1 * target_bboxes[:, 1]
        zx_flip_array = zx_flip_array * -1
        target_bboxes[:, 6] = np.pi - target_bboxes[:, 6]
    rot_angle = float(d["rot_angle"])                                     # a Python float, as np.random.random() gives
    c, s = np.cos(rot_angle), np.sin(rot_angle)
    rot_mat = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    point_cloud[:, 0:3] = np.dot(point_cloud[:, 0:3], np.transpose(rot_mat))
    point_cloud_rgb[:, 0:3] = np.dot(point_cloud_rgb[:, 0:3], np.transpose(rot_mat))
    target_bboxes[:, 0:3] = np.dot(target_bboxes[:, 0:3], np.transpose(rot_mat))
    rot_array = np.linalg.inv(np.transpose(rot_mat))
    target_bboxes[:, 6] -= rot_angle
    scale_ratio = np.expand_dims(np.tile(float(d["scale"]), 3), 0)
    scale_array = 1.0 / scale_ratio
    point_cloud[:, 0:3] *= scale_ratio
    point_cloud_rgb[:, 0:3] *= scale_ratio
    target_bboxes[:, 0:3] *= scale_ratio
    target_bboxes[:, 3:6] *= scale_ratio
    # labels (:608-700)
    raw_sizes = target_bboxes[:, 3:6] * 2 * mask[..., None]
    raw_angles = target_bboxes[:, 6] * -1 * mask
    angle_classes = np.zeros(max_num_obj, np.int64)
    angle_residuals = np.zeros(max_num_obj, np.float32)
    for i in range(k):
        angle_classes[i], angle_residuals[i] = _angle2class(raw_angles[i])
    angle_classes = angle_classes * mask
    angle_residuals = angle_residuals * mask
    dmin, dmax = point_cloud.min(axis=0)[:3], point_cloud.max(axis=0)[:3]
    centers = target_bboxes[:, 0:3]
    one, zero = np.ones((1, 3), np.float32), np.zeros((1, 3), np.float32)
    centers_n = (((centers[None] - dmin[None, None]) * (one - zero)[:, None]) / (dmax - dmin)[None, None]
                 + zero[:, None])[0] * mask[..., None]
    sizes_n = raw_sizes * (1.0 / (dmax - dmin))[None]
    return {
        "point_clouds": point_cloud.astype(np.float32),
        "point_clouds_rgb": point_cloud_rgb.astype(np.float32),
        "pcl_color": pcl_color,
        "gt_box_corners": corners_camera(centers, raw_sizes, raw_angles).astype(np.float32),
        "gt_box_corners_xyz": corners_xyz(centers, raw_sizes, raw_angles).astype(np.float32),
        "gt_box_centers": centers.astype(np.float32),
        "gt_box_centers_normalized": centers_n.astype(np.float32),
        "gt_angle_class_label": angle_classes.astype(np.int64),
        "gt_angle_residual_label": angle_residuals.astype(np.float32),
        "gt_box_sem_cls_label": np.zeros(max_num_obj, np.int64),
        "gt_box_present": mask,
        "gt_box_sizes": raw_sizes.astype(np.float32),
        "gt_box_sizes_normalized": sizes_n.astype(np.float32),
        "gt_box_angles": raw_angles.astype(np.float32),
        "point_cloud_dims_min": dmin.astype(np.float32),
        "point_cloud_dims_max": dmax.astype(np.float32),
        "input_image": img,
        "x_offset": xo, "y_offset": yo, "ori_width": frame.shape[1], "ori_height": frame.shape[0],
        "flip_array": flip_array, "zx_flip_array": zx_flip_array, "scale_array": scale_array, "rot_array": rot_array,
        "rot_angle": rot_angle, "image_flip_array": np.zeros(1) if d["image_flip"] else np.ones(1),
        "flip_length": image_size[0],
        "chosen": chosen, "box_keep": keep, "list_pos": j, "choice": choice, "count": len(rows),
    }
