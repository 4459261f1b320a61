"""Writes tests/golden/scannet_data_ref.npz: the reference's own, unmodified ScanNet training item
(datasets/scannet_anonymous_aligned_image.py ScannetDetectionAlignedImageAnonymousDataset.__getitem__, imported through
_reference_harness) for the cases of tests/scannet_data_common.py, with every np.random draw replayed from the draws
the device layer takes:

  * np.random.random()      image flip, the two point-cloud flips (0.75 = flip, 0.25 = none), rotation and scale
                            uniforms; random(3) the gain / shift uniforms; random((H, W)) the jitter uniforms of
                            the device's hash (tests/scannet_item_ref.py image_jitter_u)
  * np.random.rand(3)       RandomCuboid's crop range per attempt, (crop_range - 0.5) * 2 (exact)
  * np.random.choice(n)     RandomCuboid's centre point, data_ref.center_index(center_u, n)
  * np.random.choice(m, N)  random_sampling's rows: the positions the device's Feistel sampler picks
                            (scannet_item_ref.sample_positions)

Scene files (`_pc.npy`, `_bbox.npy`, `.jpg`, pose and intrinsic text) are written to a temporary directory; the frame
the tests use is the jpg as cv2 decodes it, in RGB.  The dataset object is built with object.__new__ and the
attributes its __init__ sets (the split file listing and the glob over the data directory are the only parts of
__init__ skipped: data_names is set to the case's scene directly).

    python tests/golden/make_scannet_data_golden.py        (needs the reference checkout and cv2)
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
import scannet_data_common as C  # noqa: E402

KEYS = ["point_clouds", "point_clouds_rgb", "pcl_color", "gt_box_corners", "gt_box_corners_xyz", "gt_box_centers",
        "gt_box_centers_normalized", "gt_angle_class_label", "gt_angle_residual_label", "gt_box_sem_cls_label",
        "gt_box_present", "gt_box_sizes", "gt_box_sizes_normalized", "gt_box_angles", "point_cloud_dims_min",
        "point_cloud_dims_max", "input_image", "x_offset", "y_offset", "ori_width", "ori_height", "flip_array",
        "zx_flip_array", "scale_array", "rot_array", "rot_angle", "image_flip_array", "K", "Rtilt"]


def write_scene(root, name):
    raw, bbox, frame, K, pose = C.scene(name)
    data = Path(root) / "frames"
    params = Path(root) / "matrix" / "scene0000_00"
    (params / "pose").mkdir(parents=True, exist_ok=True)
    (params / "intrinsic").mkdir(parents=True, exist_ok=True)
    data.mkdir(parents=True, exist_ok=True)
    np.save(data / "scene0000_00_7_pc.npy", raw)
    np.save(data / "scene0000_00_7_bbox.npy", bbox)
    cv2.imwrite(str(data / "scene0000_00_7.jpg"), cv2.cvtColor(frame, cv2.COLOR_RGB2BGR))
    # load_txt reads the 16 numbers column-major (order='F')
    np.savetxt(params / "pose" / "7.txt", pose.T.reshape(4, 4))
    np.savetxt(params / "intrinsic" / "intrinsic_color.txt", K.T.reshape(4, 4))
    decoded = cv2.cvtColor(cv2.imread(str(data / "scene0000_00_7.jpg")), cv2.COLOR_BGR2RGB)
    return str(data), str(Path(root) / "matrix"), decoded


def main():
    mod = H.load("datasets.scannet_anonymous_aligned_image")
    rc = H.load("utils.random_cuboid")
    args = types.SimpleNamespace(image_size_width=C.IMAGE_SIZE[0], image_size_height=C.IMAGE_SIZE[1],
                                 train_range_list=C.SELECT_RANGE, test_range_list=C.SELECT_RANGE)
    cfg = mod.ScannetAnonymousAlignedImageDatasetConfig(args=args)
    out = {}
    rnd = mod.np.random
    saved = rnd.random, rnd.rand, rnd.choice
    for name, (n, min_points, hw, *_rest) in C.CASES.items():
        p = C.draws(name)
        with tempfile.TemporaryDirectory() as tmp:
            data_path, param_path, decoded = write_scene(tmp, name)
            ds = object.__new__(mod.ScannetDetectionAlignedImageAnonymousDataset)
            ds.dataset_config, ds.data_path, ds.data_names = cfg, data_path, ["scene0000_00_7"]
            ds.select_range_list = np.array(C.SELECT_RANGE)
            ds.num_points, ds.use_color, ds.use_height, ds.augment, ds.image_augment = C.NUM_POINTS, False, False, True, True
            ds.use_random_cuboid = True
            ds.random_cuboid_augmentor = rc.RandomCuboid(min_points=min_points)
            ds.center_normalizing_range = [np.zeros((1, 3), dtype=np.float32), np.ones((1, 3), dtype=np.float32)]
            ds.if_input_image, ds.image_size, ds.if_padding_image = True, list(C.IMAGE_SIZE), True
            ds.param_path = param_path
            W, H_ = C.IMAGE_SIZE
            floats = [0.75 if p["image_flip"][0] else 0.25, p["image_gain_u"][0], p["image_shift_u"][0],
                      scannet_item_ref.image_jitter_u(int(p["image_seed"][0]), H_, W),
                      0.75 if p["flip_yz"][0] < 0 else 0.25, 0.75 if p["flip_xz"][0] < 0 else 0.25,
                      float(p["rot_u"][0]), float(p["scale_u"][0])]
            state = {"rand": -1}

            def random(size=None):
                v = floats.pop(0)
                assert (size is None) == np.isscalar(v), (size, v)
                return float(v) if size is None else np.array(v, np.float64).reshape(size)

            def rand(*shape):
                state["rand"] += 1
                return (p["crop_range"][0, state["rand"]] - 0.5) * 2.0

            def choice(a, size=None, replace=True):
                if size is None:
                    return data_ref.center_index(p["center_u"][0, state["rand"]], a)
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
    np.savez_compressed(HERE / "scannet_data_ref.npz", **out)


if __name__ == "__main__":
    main()
