"""The ScanNet item's CPU restatement (tests/scannet_item_ref.py scannet_item) against the reference's own
__getitem__ fed the same draws (tests/golden/scannet_data_ref.npz, tests/golden/make_scannet_data_golden.py).

Integers are exact: RandomCuboid's chosen attempt, the kept boxes, the sampled rows and positions, the angle classes.
The point rows, extents and labels are bit-exact too: the restatement performs the reference's statements on the same
operand types.  The image is the device's float32 formula (coda_image_augment) where the reference computes in
float64 (uint8 / 255.0); the two agree byte for byte except where the float64 value v * 255 lies within float32
rounding (a few 1e-5 of a level: five float32 roundings of values <= 1.05, ~6e-8 relative each, times 255) of an
integer, where truncation may land one level apart."""
from pathlib import Path

import numpy as np
import pytest

import scannet_item_ref
import scannet_data_common as C

GOLDEN = Path(__file__).resolve().parent / "golden" / "scannet_data_ref.npz"
EXACT = ["point_clouds", "point_clouds_rgb", "pcl_color", "gt_box_centers", "gt_box_centers_normalized",
         "gt_angle_class_label", "gt_angle_residual_label", "gt_box_sem_cls_label", "gt_box_present", "gt_box_sizes",
         "gt_box_sizes_normalized", "gt_box_angles", "point_cloud_dims_min", "point_cloud_dims_max", "gt_box_corners",
         "gt_box_corners_xyz", "x_offset", "y_offset", "ori_width", "ori_height", "flip_array", "zx_flip_array",
         "scale_array", "rot_array", "rot_angle", "image_flip_array"]


def item(name, frame):
    raw, bbox, _, _, _ = C.scene(name)
    _, min_points, *_ = C.CASES[name]
    return scannet_item_ref.scannet_item(raw, bbox, frame, C.draws(name), 0, C.SELECT_RANGE, C.IMAGE_SIZE,
                                         num_points=C.NUM_POINTS, min_points=min_points)


@pytest.mark.parametrize("name", list(C.CASES))
def test_scannet_item_restatement_equals_reference(name):
    g = np.load(GOLDEN)
    ref = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
    got = item(name, ref["frame"])
    for k in EXACT:
        assert np.array_equal(np.asarray(got[k]), ref[k]), k
        assert np.asarray(got[k]).dtype == ref[k].dtype or k in ("x_offset", "y_offset", "ori_width", "ori_height",
                                                                 "rot_angle"), k
    # the sampled rows are the raw rows `choice`; the rgb rows the raw rows at the crop's positions
    raw = C.scene(name)[0]
    n, min_points, _, fyz, fxz, selected, _ = C.CASES[name]
    # rotation about the up axis keeps z: z' = float32(z * scale) of the raw row `choice`
    z = (raw[got["choice"], 2].astype(np.float64) * float(C.draws(name)["scale"][0])).astype(np.float32)
    assert np.array_equal(z, ref["point_clouds"][:, 2])
    assert (n < C.NUM_POINTS) <= (got["count"] < C.NUM_POINTS)
    assert np.array_equal(raw[got["list_pos"], 3:6], ref["pcl_color"])
    chosen = got["chosen"]
    assert int(ref["rand_calls"]) == (chosen + 1 if chosen >= 0 else 100)
    if name in ("no_crop_qualifies", "fewer_points_than_samples"):      # min_points above every crop: whole scene
        assert chosen == -1 and np.array_equal(got["list_pos"], got["choice"])
    else:
        assert chosen >= 0
    if not selected:
        assert ref["gt_box_present"].sum() == 0
    else:
        assert ref["gt_box_present"].sum() == got["box_keep"].sum() > 0
    assert float(ref["flip_array"][0]) == fyz and float(ref["zx_flip_array"][0]) == fxz
    if got["count"] < C.NUM_POINTS:
        assert len(np.unique(got["list_pos"])) < C.NUM_POINTS          # with replacement
    else:
        assert len(np.unique(got["list_pos"])) == C.NUM_POINTS
    # image: bytes equal except one level at truncation boundaries of the float64 arithmetic
    img, r = got["input_image"].astype(np.int64), ref["input_image"].astype(np.int64)
    diff = np.abs(img - r)
    assert diff.max() <= 1
    assert (diff > 0).mean() < 1e-3, (diff > 0).sum()


def test_scannet_golden_covers_the_edges():
    g = np.load(GOLDEN)
    offs = {(int(g[f"{n}/x_offset"]), int(g[f"{n}/y_offset"])) for n in C.CASES}
    assert (0, 0) in offs and any(o != (0, 0) for o in offs)          # frames equal to and smaller than the canvas
    flips = {(float(g[f"{n}/flip_array"][0]), float(g[f"{n}/zx_flip_array"][0])) for n in C.CASES}
    assert flips == {(1.0, 1.0), (-1.0, -1.0), (-1.0, 1.0), (1.0, -1.0)}
    assert {int(g[f"{n}/image_flip_array"][0]) for n in C.CASES} == {0, 1}


def test_scannet_item_refuses_too_many_boxes():
    raw, bbox, frame, _, _ = C.scene("crop_both_flips_small_frame")
    many = np.repeat(bbox[:1], 65, axis=0)
    many[:, 7] = 2
    with pytest.raises(ValueError, match="max_num_obj"):
        scannet_item_ref.scannet_item(raw, many, frame, C.draws("crop_both_flips_small_frame"), 0,
                                      C.SELECT_RANGE, C.IMAGE_SIZE, num_points=C.NUM_POINTS, min_points=1500)
