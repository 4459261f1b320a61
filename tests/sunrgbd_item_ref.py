"""TEST INFRASTRUCTURE (checker only; nothing in the package imports this).

CPU restatement, in numpy, of the SUN RGB-D training item the device data layer builds (DeviceSunrgbdAugmentor in
coda_neurips2023_b200/datasets/device_pipeline.py, include/coda_data.h): datasets/sunrgbd_anonymous_aligned_image.py
:383-900 with the train split, augmentation, RandomCuboid, image input and image augmentation on.  The scene is
float64 (`_pc.npz` / `_bbox.npy`), and so is every point and box step up to the final float32 casts.  The random
draws come from the table the device takes (draw_augmentation_sunrgbd).  RandomCuboid is data_ref's, the sampler
positions, jitter and padding scannet_item_ref's.  tests/golden/sunrgbd_data_ref.npz pins it to the reference's own
__getitem__ fed those draws (tests/test_sunrgbd_data_cpu.py).
"""
from __future__ import annotations

import numpy as np

from data_ref import image_augment, random_cuboid
from scannet_item_ref import corners_camera, corners_xyz, pad_image, sample_positions

NUM_ANGLE_BIN = 12


def rotz(t):
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def angle2class(angle):                       # the dataset config's angle2class, on a float64 scalar
    angle = angle % (2 * np.pi)
    per = 2 * np.pi / float(NUM_ANGLE_BIN)
    shifted = (angle + per / 2) % (2 * np.pi)
    cls = int(shifted / per)
    return cls, shifted - (cls * per + per / 2)


def box_center(center, size, heading):
    """centre of the axis-aligned box around my_compute_box_3d's corners: rotz(-heading) @ corners, then (min + max) / 2"""
    l, w, h = size
    corners = np.dot(rotz(-1 * heading), np.vstack([[-l, l, l, -l, -l, l, l, -l], [w, w, -w, -w, w, w, -w, -w],
                                                     [h, h, h, h, -h, -h, -h, -h]]))
    corners = corners + np.asarray(center).reshape(3, 1)
    return (corners.min(axis=1) + corners.max(axis=1)) / 2


def sunrgbd_item(raw, bbox, frame, K, Rtilt, draws, b, train_range, image_size, nqueries, num_points=20000,
                 min_points=30000, max_num_obj=64):
    """The SUN RGB-D training item of scene b of `draws` (device_pipeline.draw_augmentation_sunrgbd):
    raw (n, 6) float64 `_pc.npz` rows; bbox (g, 8) float64 `_bbox.npy` rows; frame (h, w, 3) uint8 RGB;
    K / Rtilt (3, 3); train_range (min, max); image_size (W, H).  -> the reference's ret_dict fields (strings and
    uv_2d aside) plus `chosen` (RandomCuboid attempt or -1), `box_keep` and `choice` (sampled raw rows)."""
    d = {k: np.asarray(v)[b] for k, v in draws.items()}
    canvas, xo, yo = pad_image(frame, image_size)
    img = image_augment(canvas, bool(d["image_flip"]), d["image_gain"], d["image_shift"], int(d["image_seed"]))
    # train-range filter: class column 0, the raw class kept as the seen class (:476-499)
    sel = np.isin(bbox[:, 7], np.arange(train_range[0], train_range[1]))
    boxes = bbox[sel].astype(np.float64)
    seen = boxes[:, 7].copy()
    boxes[:, 7] = 0
    if len(boxes) > max_num_obj:
        raise ValueError(f"{len(boxes)} boxes after the class filter; max_num_obj is {max_num_obj}")
    pc = raw.astype(np.float64)
    xyz = pc[:, 0:3]                                          # a view: the augmentation writes through to pc
    flip_array = np.ones(1)
    if d["flip"] < 0:
        xyz[:, 0] = -1 * xyz[:, 0]
        boxes[:, 0] = -1 * boxes[:, 0]
        boxes[:, 6] = np.pi - boxes[:, 6]
        flip_array = flip_array * -1
    rot_angle = float(d["rot_angle"])
    rot_mat = rotz(rot_angle)
    xyz[:, 0:3] = np.dot(xyz[:, 0:3], np.transpose(rot_mat))
    boxes[:, 0:3] = np.dot(boxes[:, 0:3], np.transpose(rot_mat))
    rot_array = np.linalg.inv(np.transpose(rot_mat))
    boxes[:, 6] -= rot_angle
    scale_ratio = np.expand_dims(np.tile(float(d["scale"]), 3), 0)
    scale_array = 1.0 / scale_ratio
    xyz[:, 0:3] *= scale_ratio
    boxes[:, 0:3] *= scale_ratio
    boxes[:, 3:6] *= scale_ratio
    chosen, crop, keep = random_cuboid(xyz, boxes, d["crop_range"], d["center_u"], min_points, aspect=0.75)
    if chosen >= 0:
        rows = np.nonzero(np.all(xyz <= crop[3:], axis=1) & np.all(xyz >= crop[:3], axis=1))[0]
    else:
        rows = np.arange(len(xyz))
    kept, seen = boxes[keep], seen[keep]
    k = len(kept)
    # labels (:719-811)
    mask = np.zeros(max_num_obj)
    mask[:k] = 1
    raw_sizes = np.zeros((max_num_obj, 3), np.float32)
    angle_classes = np.zeros(max_num_obj, np.float32)
    angle_residuals = np.zeros(max_num_obj, np.float32)
    centers = np.zeros((max_num_obj, 3))
    for i in range(k):
        raw_sizes[i] = kept[i, 3:6] * 2
        angle_classes[i], angle_residuals[i] = angle2class(kept[i, 6])
        centers[i] = box_center(kept[i, 0:3], kept[i, 3:6], kept[i, 6])
    choice = rows[sample_positions(len(rows), int(d["seed"]), num_points)]
    point_cloud = xyz[choice]
    dmin, dmax = point_cloud.min(axis=0), point_cloud.max(axis=0)
    sizes_n = raw_sizes * (1.0 / (dmax - dmin))[None]
    box_centers = centers.astype(np.float32)
    one, zero = np.ones((1, 3), np.float32), np.zeros((1, 3), np.float32)
    centers_n = (((box_centers[None] - dmin[None, None]) * (one - zero)[:, None]) / (dmax - dmin)[None, None]
                 + zero[:, None])[0] * mask[..., None]
    angle_classes = angle_classes.astype(np.int64)
    raw_angles = angle_classes * (2 * np.pi / float(NUM_ANGLE_BIN)) + angle_residuals
    raw_angles[raw_angles > np.pi] -= 2 * np.pi
    angles32 = raw_angles.astype(np.float32)
    seen_cls = np.zeros(max_num_obj, np.int64)
    seen_cls[:k] = seen
    image_class_label = np.zeros(train_range[1])
    for i in range(k):
        if seen_cls[i] < train_range[1]:
            image_class_label[seen_cls[i]] = 1
    return {
        "point_clouds": point_cloud.astype(np.float32),
        "point_clouds_rgb": pc.astype(np.float32),
        "gt_box_corners": corners_camera(box_centers, raw_sizes, angles32).astype(np.float32),
        "gt_box_corners_xyz": corners_xyz(box_centers, raw_sizes, -angles32).astype(np.float32),
        "gt_box_centers": box_centers,
        "gt_box_centers_normalized": centers_n.astype(np.float32),
        "gt_image_class_label": image_class_label.astype(np.int64),
        "gt_box_sem_cls_label": np.zeros(max_num_obj, np.int64),
        "gt_box_seen_sem_cls_label": seen_cls,
        "gt_box_present": mask.astype(np.float32),
        "discovery_novel": np.zeros(nqueries),
        "gt_box_sizes": raw_sizes,
        "gt_box_sizes_normalized": sizes_n.astype(np.float32),
        "gt_box_angles": angles32,
        "gt_angle_class_label": angle_classes,
        "gt_angle_residual_label": angle_residuals,
        "point_cloud_dims_min": dmin,
        "point_cloud_dims_max": dmax,
        "K": np.asarray(K, np.float64), "Rtilt": np.asarray(Rtilt, np.float64),
        "input_image": img, "x_offset": xo, "y_offset": yo, "trans_mtx": np.eye(2, 2),
        "ori_width": frame.shape[1], "ori_height": frame.shape[0],
        "flip_array": flip_array, "scale_array": scale_array, "rot_array": rot_array,
        "image_flip_array": np.zeros(1) if d["image_flip"] else np.ones(1), "flip_length": image_size[0],
        "chosen": chosen, "box_keep": keep, "choice": choice, "count": len(rows),
    }
