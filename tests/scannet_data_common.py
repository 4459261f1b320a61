"""Scenes, frames and draws of the ScanNet data-layer cases, shared by tests/golden/make_scannet_data_golden.py (the
reference's __getitem__) and the tests that compare the restatement (tests/scannet_item_ref.py scannet_item) and the
device layer (DeviceScanNetAugmentor) with it."""
import numpy as np

from coda_neurips2023_b200 import synthetic
from coda_neurips2023_b200.datasets import draw_augmentation_scannet

SELECT_RANGE = [2, 4, 5, 6, 7, 8, 9, 10]               # class ids the train split keeps (train_range_list)
NUM_POINTS = 2000
IMAGE_SIZE = (64, 48)                                   # (W, H) canvas of the golden cases
# name -> (points in the raw scene, RandomCuboid min_points, frame (h, w), flip_yz, flip_xz, boxes of selected
#          classes?, seed)
CASES = {
    "crop_both_flips_small_frame": (6000, 1500, (40, 50), -1, -1, True, 0),
    "no_crop_qualifies": (5000, 4990, (48, 64), 1, 1, True, 1),
    "no_gt_after_class_filter": (6000, 1500, (31, 57), -1, 1, False, 2),
    "fewer_points_than_samples": (1500, 1400, (48, 64), 1, -1, True, 3),
    "frame_equals_canvas_yz_flip": (5000, 1000, (48, 64), -1, 1, True, 4),
    "xz_flip_only": (5500, 2000, (45, 61), 1, -1, True, 5),
}


def scene(name):
    """-> raw (n, 6) float32 [x, y, z, r, g, b], bbox rows (g, 8) float32, frame (h, w, 3) uint8 RGB,
    K (4, 4), pose (4, 4)"""
    n, _, (h, w), _, _, selected, seed = CASES[name]
    rng = np.random.default_rng(1000 + seed)
    raw = np.zeros((n, 6), np.float32)
    raw[:, 0:3] = synthetic.point_clouds(1, n, seed=seed)[0]
    raw[:, 3:6] = rng.integers(0, 256, size=(n, 3)).astype(np.float32)
    g = 9
    bbox = np.zeros((g, 8), np.float32)
    bbox[:, 0:3] = raw[rng.integers(0, n, size=g), 0:3] + rng.uniform(-0.2, 0.2, size=(g, 3))
    bbox[:, 3:6] = rng.uniform(0.1, 0.8, size=(g, 3))
    bbox[:, 6] = rng.uniform(-3, 3, size=g)
    bbox[:, 7] = rng.choice([2, 5, 7, 10, 3, 11, 13], size=g) if selected else rng.choice([3, 11, 13], size=g)
    frame = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    K = np.array([[1170.0, 0, 647.7, 0], [0, 1170.0, 483.8, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    c, s = np.cos(0.4 + seed), np.sin(0.4 + seed)
    pose = np.array([[c, 0.1 * s, -s, 1.5], [s, 0.1 * c, c, 2.0], [0, -1.0, 0.1, 1.4], [0, 0, 0, 1]])
    return raw, bbox, frame, K, pose


def draws(name):
    """the case's draws (one scene), flips forced to the case's"""
    _, _, _, fyz, fxz, _, seed = CASES[name]
    p = draw_augmentation_scannet(np.random.default_rng(2000 + seed), 1)
    p["flip_yz"], p["flip_xz"] = np.array([fyz], np.float32), np.array([fxz], np.float32)
    p["image_flip"] = np.array([seed % 2], np.uint8)
    return p
