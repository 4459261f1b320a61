"""The SUN RGB-D item's CPU restatement (tests/sunrgbd_item_ref.py sunrgbd_item) against the reference's own
__getitem__ fed the same draws (tests/golden/sunrgbd_data_ref.npz, tests/golden/make_sunrgbd_data_golden.py).

Every field is bit-exact, dtypes included, except the image: as for ScanNet (tests/test_scannet_data_cpu.py), the
restatement and the device use the float32 augmentation formula where the reference computes in float64, so a byte
may land one level apart where v * 255 lies within float32 rounding of an integer."""
from pathlib import Path

import numpy as np
import pytest

import sunrgbd_item_ref
import sunrgbd_data_common as C

GOLDEN = Path(__file__).resolve().parent / "golden" / "sunrgbd_data_ref.npz"
EXACT = ["point_clouds", "point_clouds_rgb", "gt_box_corners", "gt_box_corners_xyz", "gt_box_centers",
         "gt_box_centers_normalized", "gt_image_class_label", "gt_box_sem_cls_label", "gt_box_seen_sem_cls_label",
         "gt_box_present", "discovery_novel", "gt_box_sizes", "gt_box_sizes_normalized", "gt_box_angles",
         "gt_angle_class_label", "gt_angle_residual_label", "point_cloud_dims_min", "point_cloud_dims_max", "K",
         "Rtilt", "trans_mtx", "flip_array", "scale_array", "rot_array", "image_flip_array"]
PLAIN_INTS = ["x_offset", "y_offset", "ori_width", "ori_height", "flip_length"]


def item(name, frame):
    raw, bbox, _, K, Rtilt = C.scene(name)
    _, min_points, *_ = C.CASES[name]
    return sunrgbd_item_ref.sunrgbd_item(raw, bbox, frame, K, Rtilt, C.draws(name), 0, C.TRAIN_RANGE, C.IMAGE_SIZE,
                                         C.NQUERIES, num_points=C.NUM_POINTS, min_points=min_points)


@pytest.mark.parametrize("name", list(C.CASES))
def test_sunrgbd_item_restatement_equals_reference(name):
    g = np.load(GOLDEN)
    ref = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
    got = item(name, ref["frame"])
    for k in EXACT:
        assert np.array_equal(got[k], ref[k]), k
        assert np.asarray(got[k]).dtype == ref[k].dtype, (k, np.asarray(got[k]).dtype, ref[k].dtype)
    for k in PLAIN_INTS:
        assert int(got[k]) == int(ref[k]), k
    n, _, _, flip, _, boxes, _ = C.CASES[name]
    chosen = got["chosen"]
    assert int(ref["rand_calls"]) == (chosen + 1 if chosen >= 0 else 100)
    if name in ("no_crop_qualifies", "fewer_points_than_samples"):      # min_points above every crop: whole scene
        assert chosen == -1 and got["count"] == n
    else:
        assert chosen >= 0 and got["count"] < n
    present = int(ref["gt_box_present"].sum())
    assert (present > 0) == (boxes == "train")
    if boxes == "train":
        assert ref["gt_image_class_label"].sum() > 0
        assert set(ref["gt_box_seen_sem_cls_label"][:present]) <= set(range(*C.TRAIN_RANGE))
    assert float(ref["flip_array"][0]) == flip
    # point_clouds_rgb is the whole raw scene, transformed and not cropped; its colours are the raw ones
    raw = C.scene(name)[0]
    assert ref["point_clouds_rgb"].shape == (n, 6)
    assert np.array_equal(ref["point_clouds_rgb"][:, 3:6], raw[:, 3:6].astype(np.float32))
    assert ref["point_cloud_dims_min"].dtype == np.float64
    img, r = got["input_image"].astype(np.int64), ref["input_image"].astype(np.int64)
    diff = np.abs(img - r)
    assert diff.max() <= 1
    assert (diff > 0).mean() < 1e-3, (diff > 0).sum()


def test_sunrgbd_golden_covers_the_edges():
    g = np.load(GOLDEN)
    offs = {(int(g[f"{n}/x_offset"]), int(g[f"{n}/y_offset"])) for n in C.CASES}
    assert (0, 0) in offs and any(o != (0, 0) for o in offs)          # frames equal to and smaller than the canvas
    assert {float(g[f"{n}/flip_array"][0]) for n in C.CASES} == {1.0, -1.0}
    assert {int(g[f"{n}/image_flip_array"][0]) for n in C.CASES} == {0, 1}
    assert any(int(g[f"{n}/rand_calls"]) == 100 for n in C.CASES)       # no crop qualifies
    assert str(g["numpy_version"])


def test_sunrgbd_item_refuses_too_many_boxes():
    raw, bbox, frame, K, Rtilt = C.scene("crop_flip_small_frame")
    many = np.repeat(bbox[:1], 65, axis=0)
    many[:, 7] = 3
    with pytest.raises(ValueError, match="max_num_obj"):
        sunrgbd_item_ref.sunrgbd_item(raw, many, frame, K, Rtilt, C.draws("crop_flip_small_frame"), 0, C.TRAIN_RANGE,
                                      C.IMAGE_SIZE, C.NQUERIES, num_points=C.NUM_POINTS, min_points=1500)
