"""The ScanNet item on the device (DeviceScanNetAugmentor, include/coda_data.h) against its CPU restatement
tests/scannet_item_ref.py scannet_item (pinned to the reference's __getitem__ by tests/test_scannet_data_cpu.py): bit
for bit at the golden's edge cases and at the training shape; the batch's inverse arrays undo its own augmentation in the
ScanNet projection; one training step on such a batch."""
import warnings

import numpy as np
import pytest
import torch

import scannet_item_ref
import scannet_data_common as C
from coda_neurips2023_b200 import ops, synthetic
from coda_neurips2023_b200.datasets import DeviceScanNetAugmentor, draw_augmentation_scannet
from coda_neurips2023_b200.datasets.device_pipeline import identity_draws_scannet

pytestmark = pytest.mark.gpu

BITS = ["point_clouds", "point_clouds_rgb", "pcl_color", "gt_box_centers", "gt_box_centers_normalized",
        "gt_angle_class_label", "gt_angle_residual_label", "gt_box_sem_cls_label", "gt_box_present", "gt_box_sizes",
        "gt_box_sizes_normalized", "gt_box_angles", "point_cloud_dims_min", "point_cloud_dims_max", "input_image",
        "x_offset", "y_offset", "ori_width", "ori_height", "flip_array", "zx_flip_array", "scale_array", "rot_array",
        "rot_angle", "image_flip_array"]
# corners: cos / sin of the float32 heading are the device's cosf / sinf and numpy's float32 routines, each within
# about an ulp (6e-8) of the true value; times box half-sizes below 2 m plus one float32 rounding of a coordinate
# below 10 m: 1e-6 absolute
CORNER_ATOL = 1e-6


def run_device(scenes, draws, aug, K=None, pose=None):
    b = len(scenes)
    nmax = max(len(s[0]) for s in scenes)
    gmax = max(len(s[1]) for s in scenes)
    pts = np.zeros((b, nmax, 6), np.float32)
    boxes = np.zeros((b, gmax, 8), np.float32)
    for i, s in enumerate(scenes):
        pts[i, :len(s[0])] = s[0]
        boxes[i, :len(s[1])] = s[1]
    npts = torch.tensor([len(s[0]) for s in scenes], dtype=torch.int32).cuda()
    nbox = torch.tensor([len(s[1]) for s in scenes], dtype=torch.int32).cuda()
    frames = [torch.from_numpy(s[2]).cuda() for s in scenes]
    K = np.stack([s[3] for s in scenes]) if K is None else K
    pose = np.stack([s[4] for s in scenes]) if pose is None else pose
    return aug.batch(torch.from_numpy(pts).cuda(), npts, torch.from_numpy(boxes).cuda(), nbox, frames, K, pose, draws)


def compare(got, b, scene, draws, min_points, num_points, image_size):
    exp = scannet_item_ref.scannet_item(scene[0], scene[1], scene[2], draws, b, C.SELECT_RANGE, image_size,
                                        num_points=num_points, min_points=min_points)
    for k in BITS:
        g = got[k][b].cpu().numpy()
        e = np.asarray(exp[k]).reshape(g.shape)
        assert np.array_equal(g, e), k
    for k in ("gt_box_corners", "gt_box_corners_xyz"):
        assert np.abs(got[k][b].cpu().numpy() - exp[k]).max() <= CORNER_ATOL, k
    return exp


@pytest.mark.parametrize("name", list(C.CASES))
def test_device_item_equals_restatement_at_the_golden_cases(built_lib, name):
    _, min_points, *_ = C.CASES[name]
    aug = DeviceScanNetAugmentor(C.SELECT_RANGE, num_points=C.NUM_POINTS, random_cuboid_min_points=min_points,
                                 image_size=C.IMAGE_SIZE)
    scene = C.scene(name)
    draws = C.draws(name)
    got = run_device([scene], draws, aug)
    compare(got, 0, scene, draws, min_points, C.NUM_POINTS, C.IMAGE_SIZE)


def _big_scenes(batch, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(batch):
        n = int(rng.integers(50000, 150001))
        raw = np.zeros((n, 6), np.float32)
        raw[:, 0:3] = synthetic.point_clouds(1, n, seed=seed * 100 + i)[0]
        raw[:, 3:6] = rng.integers(0, 256, size=(n, 3))
        g = int(rng.integers(0, 40))
        bbox = np.zeros((g, 8), np.float32)
        bbox[:, 0:3] = raw[rng.integers(0, n, size=g), 0:3]
        bbox[:, 3:6] = rng.uniform(0.1, 1.0, size=(g, 3))
        bbox[:, 6] = rng.uniform(-3, 3, size=g)
        bbox[:, 7] = rng.choice([2, 3, 5, 7, 11, 10], size=g)
        h, w = (968, 1296) if i % 2 == 0 else (900, 1200)
        frame = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        K = np.array([[1170.0, 0, 647.7, 0], [0, 1170.0, 483.8, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
        c, s = np.cos(0.3 * i), np.sin(0.3 * i)
        pose = np.array([[c, 0.1 * s, -s, 1.5], [s, 0.1 * c, c, 2.0], [0, -1.0, 0.1, 1.4], [0, 0, 0, 1]])
        out.append((raw, bbox, frame, K, pose))
    return out


def test_device_batch_equals_restatement_at_the_training_shape(built_lib):
    scenes = _big_scenes(8, 1)
    draws = draw_augmentation_scannet(np.random.default_rng(5), 8)
    aug = DeviceScanNetAugmentor(C.SELECT_RANGE)
    got = run_device(scenes, draws, aug)
    assert tuple(got["point_clouds"].shape) == (8, 40000, 3) and tuple(got["input_image"].shape) == (8, 968, 1296, 3)
    chosen = 0
    for b in range(8):
        exp = compare(got, b, scenes[b], draws, 30000, 40000, (1296, 968))
        chosen += exp["chosen"] >= 0
    print(f"SCANNET data B=8: {chosen} of 8 scenes cropped")


def test_inverse_arrays_undo_the_augmentation_in_the_scannet_projection(built_lib):
    """boxes_in_image(camera="scannet") of every kept GT box: the augmented batch and the same scenes with identity
    point-cloud draws (same crop, sampling and image) give the same fp64 image extent.  The corners are float32 in
    both batches (as the reference stores them), so the two agree to float32 rounding of the corners (a few 1e-7
    relative of a coordinate, through the projection), not to fp64: 1e-5 relative of the extent's span."""
    scenes = _big_scenes(4, 2)
    draws = draw_augmentation_scannet(np.random.default_rng(6), 4)
    draws["flip_yz"][:] = [-1, 1, -1, 1]
    draws["flip_xz"][:] = [-1, -1, 1, 1]
    aug = DeviceScanNetAugmentor(C.SELECT_RANGE)
    a = run_device(scenes, draws, aug)
    i = run_device(scenes, identity_draws_scannet(draws), aug)
    assert torch.equal(a["gt_box_present"], i["gt_box_present"])
    ea = ops.boxes_in_image(a["gt_box_corners_xyz"], a["gt_box_sizes"], a, camera="scannet", extent=True)
    ei = ops.boxes_in_image(i["gt_box_corners_xyz"], i["gt_box_sizes"], i, camera="scannet", extent=True)
    present = a["gt_box_present"].bool() & ea[1] & ei[1]
    assert int(present.sum()) > 0
    xa, xi = ea[2][present], ei[2][present]
    span = (xi[:, 2:] - xi[:, :2]).abs().max(1).values.clamp_min(1.0)
    rel = ((xa - xi).abs().max(1).values / span).max().item()
    print(f"SCANNET projection round trip: {int(present.sum())} boxes, max rel extent diff {rel:.2e}")
    assert rel <= 1e-5
    assert torch.equal(ea[1] & a["gt_box_present"].bool(), ei[1] & i["gt_box_present"].bool())


def test_one_stage1_step_on_a_device_batch_is_finite(built_lib):
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.engine import TrainStep
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(dataset_name="scannet_anonymous_aligned_image", matcher_giou_cost=2.0,
                               matcher_center_cost=0.0, matcher_objectness_cost=0.0, loss_no_object_weight=0.25,
                               base_lr=1.4142e-4, train_range_max=10, test_range_max=60, image_size_width=1296,
                               image_size_height=968, nqueries=128)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model, crit = model.cuda().train(), build_criterion(args, cfg).cuda()
    scenes = _big_scenes(2, 3)
    batch = run_device(scenes, draw_augmentation_scannet(np.random.default_rng(7), 2), DeviceScanNetAugmentor(C.SELECT_RANGE))
    step = TrainStep(args, model, crit, torch.device("cuda", 0))
    step.prepare(batch)
    np.random.seed(3)
    loss, _ = step(batch, 0.0)
    print(f"SCANNET stage-1 step on a device batch: loss {float(loss)}")
    assert np.isfinite(float(loss))


def test_refusals(built_lib):
    with pytest.raises(NotImplementedError, match="use_color"):
        DeviceScanNetAugmentor(C.SELECT_RANGE, use_color=True)
    with pytest.raises(NotImplementedError, match="use_height"):
        DeviceScanNetAugmentor(C.SELECT_RANGE, use_height=True)
    raw, bbox, frame, K, pose = C.scene("crop_both_flips_small_frame")
    many = np.repeat(bbox[:1], 65, axis=0)
    many[:, 7] = 2
    aug = DeviceScanNetAugmentor(C.SELECT_RANGE, num_points=C.NUM_POINTS, image_size=C.IMAGE_SIZE)
    with pytest.raises(ValueError, match="max_num_obj"):
        run_device([(raw, many, frame, K, pose)], C.draws("crop_both_flips_small_frame"), aug)


def test_sample_points_ex_keeps_the_bits_of_sample_points(built_lib):
    from coda_neurips2023_b200._lib import lib, ptr, stream_of
    from coda_neurips2023_b200.datasets.device_pipeline import _i
    rng = np.random.default_rng(0)
    b, nmax, nsample = 3, 7000, 3000
    pts = torch.from_numpy(rng.standard_normal((b, nmax, 6)).astype(np.float32)).cuda()
    npts = torch.tensor([7000, 2000, 5000], dtype=torch.int32).cuda()
    crop = torch.tensor([[-1.0, -1.0, -1.0, 1.0, 1.0, 1.0], [-9.0] * 3 + [9.0] * 3, [-0.5, -2, -2, 2, 2, 2]],
                        dtype=torch.float64).cuda()
    seed = torch.tensor([1, 2, 3], dtype=torch.int32).cuda()
    outs = []
    for ex in (False, True):
        lst = torch.empty((b, nmax), dtype=torch.int32).cuda()
        cnt = torch.empty((b,), dtype=torch.int32).cuda()
        out = torch.empty((b, nsample, 6)).cuda()
        ch = torch.empty((b, nsample), dtype=torch.int32).cuda()
        dims = torch.empty((b, 6)).cuda()
        st = stream_of(pts)
        if ex:
            pos = torch.empty((b, nsample), dtype=torch.int32).cuda()
            rgb = torch.empty((b, nsample, 4)).cuda()
            assert lib().coda_sample_points_ex(_i(b), _i(nmax), _i(6), _i(nsample), _i(4), ptr(npts), ptr(pts),
                                               ptr(crop), ptr(seed), ptr(lst), ptr(cnt), ptr(out), ptr(ch), ptr(pos),
                                               ptr(rgb), ptr(dims), st) == 0
            for i in range(b):
                assert torch.equal(rgb[i], pts[i, pos[i].long(), :4])
        else:
            assert lib().coda_sample_points(_i(b), _i(nmax), _i(6), _i(nsample), ptr(npts), ptr(pts), ptr(crop),
                                            ptr(seed), ptr(lst), ptr(cnt), ptr(out), ptr(ch), ptr(dims), st) == 0
        outs.append((out, ch, cnt, dims))
    for x, y in zip(*outs):
        assert torch.equal(x, y)
