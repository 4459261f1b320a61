"""Scenes, frames and draws of the SUN RGB-D data-layer cases, shared by tests/golden/make_sunrgbd_data_golden.py (the
reference's __getitem__) and the tests that compare the restatement (tests/sunrgbd_item_ref.py sunrgbd_item) and the
device layer (DeviceSunrgbdAugmentor) with it.  Scenes are float64, as the `_pc.npz` / `_bbox.npy` files are."""
import numpy as np

from coda_neurips2023_b200 import synthetic
from coda_neurips2023_b200.datasets import draw_augmentation_sunrgbd

TRAIN_RANGE = (0, 10)                                   # train_range_min, train_range_max
NQUERIES = 16
NUM_POINTS = 2000
IMAGE_SIZE = (64, 48)                                   # (W, H) canvas of the golden cases
# name -> (points in the raw scene, RandomCuboid min_points, frame (h, w), point flip, image flip, boxes: "train"
#          (some of a train class), "novel" (none of a train class) or "none" (no rows), seed)
CASES = {
    "crop_flip_small_frame": (6000, 1500, (40, 50), -1, 1, "train", 0),
    "no_crop_qualifies": (5000, 4990, (48, 64), 1, 0, "train", 1),
    "no_train_class_box": (6000, 1500, (31, 57), -1, 0, "novel", 2),
    "no_boxes": (5500, 1500, (45, 61), 1, 1, "none", 3),
    "fewer_points_than_samples": (1500, 1400, (48, 64), 1, 1, "train", 4),
    "frame_equals_canvas": (5000, 1000, (48, 64), -1, 0, "train", 5),
}


def scene(name):
    """-> raw (n, 6) float64 [x, y, z, r, g, b] (colour in 0-1), bbox rows (g, 8) float64
    [cx, cy, cz, l/2, w/2, h/2, heading, class], frame (h, w, 3) uint8 RGB, K (3, 3), Rtilt (3, 3)"""
    n, _, (h, w), _, _, boxes, seed = CASES[name]
    rng = np.random.default_rng(3000 + seed)
    raw = np.zeros((n, 6))
    raw[:, 0:3] = synthetic.point_clouds(1, n, seed=seed)[0].astype(np.float64) + rng.uniform(-1e-3, 1e-3, (n, 3))
    raw[:, 3:6] = rng.random((n, 3))
    g = {"train": 9, "novel": 6, "none": 0}[boxes]
    bbox = np.zeros((g, 8))
    bbox[:, 0:3] = raw[rng.integers(0, n, size=g), 0:3] + rng.uniform(-0.2, 0.2, size=(g, 3))
    bbox[:, 3:6] = rng.uniform(0.1, 0.8, size=(g, 3))
    bbox[:, 6] = rng.uniform(-3, 3, size=g)
    classes = [1, 3, 7, 12, 15, 20] if boxes == "train" else [10, 12, 15, 20]
    bbox[:, 7] = rng.choice(classes, size=g)
    frame = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    K = np.array([[529.5, 0.0, 365.0], [0.0, 529.5, 265.0], [0.0, 0.0, 1.0]])
    c, s = np.cos(0.05 * (seed + 1)), np.sin(0.05 * (seed + 1))
    Rtilt = np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])
    return raw, bbox, frame, K, Rtilt


def draws(name):
    """the case's draws (one scene), flips forced to the case's"""
    _, _, _, flip, image_flip, _, seed = CASES[name]
    p = draw_augmentation_sunrgbd(np.random.default_rng(4000 + seed), 1)
    p["flip"] = np.array([flip], np.float32)
    p["image_flip"] = np.array([image_flip], np.uint8)
    return p
