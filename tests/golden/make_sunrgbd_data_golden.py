"""Writes tests/golden/sunrgbd_data_ref.npz: the reference's own, unmodified SUN RGB-D training item
(datasets/sunrgbd_anonymous_aligned_image.py SunrgbdAnonymousAlignedImageDetectionDataset.__getitem__, imported through
_reference_harness) for the cases of tests/sunrgbd_data_common.py, with every np.random draw replayed from the draws
the device layer takes:

  * np.random.random()      image flip, point flip (0.75 = flip, 0.25 = none), rotation and scale uniforms;
                            random(3) the gain / shift uniforms; random((H, W)) the jitter uniforms of the device's hash
                            (tests/scannet_item_ref.py image_jitter_u)
  * np.random.rand(3)       RandomCuboid's crop-range uniforms per attempt (crop_u)
  * np.random.choice(n)     RandomCuboid's centre point, data_ref.center_index(center_u, n)
  * np.random.choice(m, N)  random_sampling's rows: the positions the device's Feistel sampler picks
                            (scannet_item_ref.sample_positions)

Scene files (float64 `_pc.npz` / `_bbox.npy`, `.jpg`, calib text) are written to a temporary directory; the frame
the tests use is the jpg as cv2 decodes it, in RGB.  The dataset object is built with object.__new__ and the
attributes its __init__ sets (the directory listing is the only part of __init__ skipped: scan_names is set to the
case's scene directly).  utils.votenet_pc_util is stubbed: it imports matplotlib.pyplot's colour maps, which the
harness stubs out, and the item only imports its unused visualisation writers.

    python tests/golden/make_sunrgbd_data_golden.py        (needs the reference checkout and cv2)
"""
import sys
import tempfile
import types
from pathlib import Path

import cv2
import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent.parent / "oracle"))
import _reference_harness as H  # noqa: E402
import data_ref  # noqa: E402
import scannet_item_ref  # noqa: E402
import sunrgbd_data_common as C  # noqa: E402

KEYS = ["point_clouds", "point_clouds_rgb", "gt_box_corners", "gt_box_corners_xyz", "gt_box_centers",
        "gt_box_centers_normalized", "gt_image_class_label", "gt_box_sem_cls_label", "gt_box_seen_sem_cls_label",
        "gt_box_present", "discovery_novel", "scan_idx", "gt_box_sizes", "gt_box_sizes_normalized", "gt_box_angles",
        "gt_angle_class_label", "gt_angle_residual_label", "point_cloud_dims_min", "point_cloud_dims_max", "K",
        "Rtilt", "input_image", "y_offset", "x_offset", "trans_mtx", "ori_width", "ori_height", "flip_array",
        "scale_array", "rot_array", "image_flip_array", "flip_length"]
SCAN = "000007"


def write_scene(root, name):
    raw, bbox, frame, K, Rtilt = C.scene(name)
    root = Path(root)
    for d in ("data_train", "calib", "image"):
        (root / d).mkdir(parents=True, exist_ok=True)
    np.savez_compressed(root / "data_train" / f"{SCAN}_pc.npz", pc=raw)
    np.save(root / "data_train" / f"{SCAN}_bbox.npy", bbox)
    cv2.imwrite(str(root / "image" / f"{SCAN}.jpg"), cv2.cvtColor(frame, cv2.COLOR_RGB2BGR))
    # the item reads each line's nine numbers column-major (order='F'): Rtilt, then K
    with open(root / "calib" / f"{SCAN}.txt", "w") as f:
        for m in (Rtilt, K):
            f.write(" ".join(repr(float(v)) for v in m.flatten(order="F")) + "\n")
    decoded = cv2.cvtColor(cv2.imread(str(root / "image" / f"{SCAN}.jpg")), cv2.COLOR_BGR2RGB)
    return str(root / "data_train"), str(root / "calib"), str(root / "image"), decoded


def main():
    H.install()
    sys.modules["utils.votenet_pc_util"] = types.SimpleNamespace(write_oriented_bbox=None, write_ply=None,
                                                                 write_ply_rgb=None)
    mod = H.load("datasets.sunrgbd_anonymous_aligned_image")
    rc = H.load("utils.random_cuboid")
    args = types.SimpleNamespace(if_use_v1=True, image_size_width=C.IMAGE_SIZE[0], image_size_height=C.IMAGE_SIZE[1],
                                 test_range_min=0, test_range_max=40, train_range_min=C.TRAIN_RANGE[0],
                                 train_range_max=C.TRAIN_RANGE[1], nqueries=C.NQUERIES)
    cfg = mod.SunrgbdAnonymousAlignedImageDatasetConfig(if_print=False, args=args)
    out = {"numpy_version": np.array(np.__version__)}
    rnd = mod.np.random
    saved = rnd.random, rnd.rand, rnd.choice
    for name, (n, min_points, *_rest) in C.CASES.items():
        p = C.draws(name)
        with tempfile.TemporaryDirectory() as tmp:
            data_path, calib_path, image_path, decoded = write_scene(tmp, name)
            ds = object.__new__(mod.SunrgbdAnonymousAlignedImageDetectionDataset)
            ds.split_set, ds.dataset_config, ds.use_v1 = "train", cfg, True
            ds.image_size, ds.if_padding_image = cfg.image_size, cfg.if_padding_image
            ds.data_path, ds.calib_path, ds.image_path = data_path, calib_path + "/", image_path + "/"
            ds.scan_names, ds.if_input_image = [SCAN], True
            ds.num_points, ds.augment, ds.image_augment = C.NUM_POINTS, True, True
            ds.use_color, ds.use_height, ds.use_random_cuboid = False, False, True
            ds.random_cuboid_augmentor = rc.RandomCuboid(min_points=min_points, aspect=0.75, min_crop=0.75,
                                                         max_crop=1.0)
            ds.center_normalizing_range = [np.zeros((1, 3), dtype=np.float32), np.ones((1, 3), dtype=np.float32)]
            ds.max_num_obj, ds.len_datasets = 64, 1
            W, H_ = C.IMAGE_SIZE
            floats = [0.75 if p["image_flip"][0] else 0.25, p["image_gain_u"][0], p["image_shift_u"][0],
                      scannet_item_ref.image_jitter_u(int(p["image_seed"][0]), H_, W),
                      0.75 if p["flip"][0] < 0 else 0.25, float(p["rot_u"][0]), float(p["scale_u"][0])]
            state = {"rand": -1}

            def random(size=None):
                v = floats.pop(0)
                assert (size is None) == np.isscalar(v), (size, v)
                return float(v) if size is None else np.array(v, np.float64).reshape(size)

            def rand(*shape):
                state["rand"] += 1
                return p["crop_u"][0, state["rand"]].copy()

            def choice(a, size=None, replace=True):
                if size is None:
                    return data_ref.center_index(p["center_u"][0, state["rand"]], a)
                assert replace == (a < size)
                return scannet_item_ref.sample_positions(a, int(p["seed"][0]), size)

            rnd.random, rnd.rand, rnd.choice = random, rand, choice
            try:
                item = ds[0]
            finally:
                rnd.random, rnd.rand, rnd.choice = saved
            assert not floats
            out[f"{name}/frame"] = decoded
            out[f"{name}/rand_calls"] = np.array(state["rand"] + 1)             # RandomCuboid attempts made
            for k in KEYS:
                out[f"{name}/{k}"] = np.asarray(item[k])
    np.savez_compressed(HERE / "sunrgbd_data_ref.npz", **out)


if __name__ == "__main__":
    main()
