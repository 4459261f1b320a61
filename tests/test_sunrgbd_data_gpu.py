"""The SUN RGB-D item on the device (DeviceSunrgbdAugmentor, include/coda_data.h) against its CPU restatement
tests/sunrgbd_item_ref.py sunrgbd_item (pinned to the reference's __getitem__ by tests/test_sunrgbd_data_cpu.py): bit
for bit, dtypes included, at the golden's edge cases and at the training shape; the batch's inverse arrays undo its own
augmentation in the SUN RGB-D projection; one training step on such a batch; the float64 entry points against the
float32 ones."""
import warnings

import numpy as np
import pytest
import torch

import sunrgbd_item_ref
import sunrgbd_data_common as C
from coda_neurips2023_b200 import ops, synthetic
from coda_neurips2023_b200.datasets import DeviceSunrgbdAugmentor, draw_augmentation_sunrgbd
from coda_neurips2023_b200.datasets.device_pipeline import identity_draws_sunrgbd

pytestmark = pytest.mark.gpu

BITS = ["point_clouds", "point_clouds_rgb", "gt_box_centers", "gt_box_centers_normalized", "gt_image_class_label",
        "gt_box_sem_cls_label", "gt_box_seen_sem_cls_label", "gt_box_present", "discovery_novel", "gt_box_sizes",
        "gt_box_sizes_normalized", "gt_box_angles", "gt_angle_class_label", "gt_angle_residual_label",
        "point_cloud_dims_min", "point_cloud_dims_max", "K", "Rtilt", "input_image", "x_offset", "y_offset",
        "trans_mtx", "ori_width", "ori_height", "flip_array", "scale_array", "rot_array", "image_flip_array",
        "flip_length"]
# corners: the float32 heading's cos / sin are the device's and numpy's float32 routines, each within about an ulp;
# the ScanNet tolerance (tests/test_scannet_data_gpu.py)
CORNER_ATOL = 1e-6
TORCH_DTYPE = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64,
               np.dtype(np.int64): torch.int64, np.dtype(np.uint8): torch.uint8}


def run_device(scenes, draws, aug):
    b = len(scenes)
    n = len(scenes[0][0])
    gmax = max(1, max(len(s[1]) for s in scenes))
    pts = np.stack([s[0] for s in scenes])
    boxes = np.zeros((b, gmax, 8))
    for i, s in enumerate(scenes):
        boxes[i, :len(s[1])] = s[1]
    npts = torch.full((b,), n, dtype=torch.int32)
    nbox = torch.tensor([len(s[1]) for s in scenes], dtype=torch.int32).cuda()
    frames = [torch.from_numpy(s[2]).cuda() for s in scenes]
    K, Rtilt = np.stack([s[3] for s in scenes]), np.stack([s[4] for s in scenes])
    return aug.batch(torch.from_numpy(pts).cuda(), npts, torch.from_numpy(boxes).cuda(), nbox, frames, K, Rtilt,
                     draws)


def compare(got, b, scene, draws, min_points, num_points, image_size, nqueries):
    exp = sunrgbd_item_ref.sunrgbd_item(scene[0], scene[1], scene[2], scene[3], scene[4], draws, b, C.TRAIN_RANGE,
                                        image_size, nqueries, num_points=num_points, min_points=min_points)
    for k in BITS:
        g = got[k][b].cpu().numpy()
        e = np.asarray(exp[k])
        if e.dtype.kind == "i" and e.ndim == 0:
            e = e.astype(np.int64)                     # default collate makes the item's Python ints int64
        assert got[k].dtype == TORCH_DTYPE[e.dtype], (k, got[k].dtype, e.dtype)
        assert np.array_equal(g, e.reshape(g.shape)), k
    for k in ("gt_box_corners", "gt_box_corners_xyz"):
        assert got[k].dtype == torch.float32
        assert np.abs(got[k][b].cpu().numpy() - exp[k]).max() <= CORNER_ATOL, k
    assert int(got["scan_idx"][b]) == b
    return exp


@pytest.mark.parametrize("name", list(C.CASES))
def test_device_item_equals_restatement_at_the_golden_cases(built_lib, name):
    _, min_points, *_ = C.CASES[name]
    aug = DeviceSunrgbdAugmentor(*C.TRAIN_RANGE, C.NQUERIES, num_points=C.NUM_POINTS,
                                 random_cuboid_min_points=min_points, image_size=C.IMAGE_SIZE)
    scene = C.scene(name)
    draws = C.draws(name)
    got = run_device([scene], draws, aug)
    compare(got, 0, scene, draws, min_points, C.NUM_POINTS, C.IMAGE_SIZE, C.NQUERIES)


def _big_scenes(batch, seed, n=50000):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(batch):
        raw = np.zeros((n, 6))
        raw[:, 0:3] = synthetic.point_clouds(1, n, seed=seed * 100 + i)[0] + rng.uniform(-1e-3, 1e-3, (n, 3))
        raw[:, 3:6] = rng.random((n, 3))
        g = int(rng.integers(0, 40))
        bbox = np.zeros((g, 8))
        bbox[:, 0:3] = raw[rng.integers(0, n, size=g), 0:3]
        bbox[:, 3:6] = rng.uniform(0.1, 1.0, size=(g, 3))
        bbox[:, 6] = rng.uniform(-3, 3, size=g)
        bbox[:, 7] = rng.choice([0, 2, 5, 9, 10, 14, 30], size=g)
        h, w = (531, 730) if i % 2 == 0 else (427, 561)
        frame = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        K = np.array([[529.5, 0.0, 365.0], [0.0, 529.5, 265.0], [0.0, 0.0, 1.0]])
        c, s = np.cos(0.02 * i), np.sin(0.02 * i)
        Rtilt = np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])
        out.append((raw, bbox, frame, K, Rtilt))
    return out


def test_device_batch_equals_restatement_at_the_training_shape(built_lib):
    scenes = _big_scenes(8, 1)
    draws = draw_augmentation_sunrgbd(np.random.default_rng(5), 8)
    aug = DeviceSunrgbdAugmentor(0, 10, 256)
    got = run_device(scenes, draws, aug)
    assert tuple(got["point_clouds"].shape) == (8, 20000, 3) and tuple(got["input_image"].shape) == (8, 531, 730, 3)
    assert tuple(got["point_clouds_rgb"].shape) == (8, 50000, 6)
    chosen = 0
    for b in range(8):
        exp = compare(got, b, scenes[b], draws, 30000, 20000, (730, 531), 256)
        chosen += exp["chosen"] >= 0
    print(f"SUNRGBD data B=8: {chosen} of 8 scenes cropped")
    assert chosen > 0


def test_inverse_arrays_undo_the_augmentation_in_the_sunrgbd_projection(built_lib):
    """boxes_in_image(camera="sunrgbd") of every kept GT box: the augmented batch and the same scenes with identity
    point-cloud draws (same crop attempts, sampling and image) give the same fp64 image extent, to the float32
    rounding of the corners both batches store (1e-5 relative of the extent's span).  RandomCuboid runs on the
    transformed cloud, so its min_points is set above every crop: both batches keep every box."""
    scenes = _big_scenes(4, 2)
    draws = draw_augmentation_sunrgbd(np.random.default_rng(6), 4)
    draws["flip"][:] = [-1, 1, -1, 1]
    aug = DeviceSunrgbdAugmentor(0, 10, 256, random_cuboid_min_points=10 ** 9)       # no crop: the same boxes
    a = run_device(scenes, draws, aug)
    i = run_device(scenes, identity_draws_sunrgbd(draws), aug)
    assert torch.equal(a["gt_box_present"], i["gt_box_present"])
    ea = ops.boxes_in_image(a["gt_box_corners_xyz"], a["gt_box_sizes"], a, camera="sunrgbd", extent=True)
    ei = ops.boxes_in_image(i["gt_box_corners_xyz"], i["gt_box_sizes"], i, camera="sunrgbd", extent=True)
    present = a["gt_box_present"].bool() & ea[1] & ei[1]
    assert int(present.sum()) > 0
    xa, xi = ea[2][present], ei[2][present]
    span = (xi[:, 2:] - xi[:, :2]).abs().max(1).values.clamp_min(1.0)
    rel = ((xa - xi).abs().max(1).values / span).max().item()
    print(f"SUNRGBD projection round trip: {int(present.sum())} boxes, max rel extent diff {rel:.2e}")
    assert rel <= 1e-5


def test_one_stage1_step_on_a_device_batch_is_finite(built_lib):
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.engine import TrainStep
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(nqueries=128)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model, crit = model.cuda().train(), build_criterion(args, cfg).cuda()
    batch = run_device(_big_scenes(2, 3), draw_augmentation_sunrgbd(np.random.default_rng(7), 2),
                       DeviceSunrgbdAugmentor(0, args.train_range_max, args.nqueries))
    step = TrainStep(args, model, crit, torch.device("cuda", 0))
    step.prepare(batch)
    np.random.seed(3)
    loss, _ = step(batch, 0.0)
    print(f"SUNRGBD stage-1 step on a device batch: loss {float(loss)}")
    assert np.isfinite(float(loss))


def test_refusals(built_lib):
    with pytest.raises(NotImplementedError, match="use_color"):
        DeviceSunrgbdAugmentor(0, 10, 16, use_color=True)
    with pytest.raises(NotImplementedError, match="use_height"):
        DeviceSunrgbdAugmentor(0, 10, 16, use_height=True)
    raw, bbox, frame, K, Rtilt = C.scene("crop_flip_small_frame")
    draws = C.draws("crop_flip_small_frame")
    aug = DeviceSunrgbdAugmentor(*C.TRAIN_RANGE, C.NQUERIES, num_points=C.NUM_POINTS, image_size=C.IMAGE_SIZE)
    frames = [torch.from_numpy(frame).cuda()]
    nb = torch.tensor([len(bbox)], dtype=torch.int32)
    with pytest.raises(TypeError, match="float64"):
        aug.batch(torch.from_numpy(raw[None].astype(np.float32)).cuda(), [len(raw)], torch.from_numpy(bbox[None]).cuda(),
                  nb, frames, K[None], Rtilt[None], draws)
    many = np.repeat(bbox[:1], 65, axis=0)
    many[:, 7] = 3
    with pytest.raises(ValueError, match="max_num_obj"):
        run_device([(raw, many, frame, K, Rtilt)], draws, aug)
    two = draw_augmentation_sunrgbd(np.random.default_rng(0), 2)
    pts = torch.from_numpy(np.stack([raw, raw])).cuda()
    with pytest.raises(ValueError, match="raw rows"):
        aug.batch(pts, [len(raw), len(raw) - 10], torch.from_numpy(np.stack([bbox, bbox])).cuda(), nb.repeat(2),
                  frames * 2, np.stack([K, K]), np.stack([Rtilt, Rtilt]), two)


def test_float64_entry_points_give_the_float32_integer_results(built_lib):
    """On coordinates that are multiples of 1/64 (exact in float32, and so are their extents), the float32 and float64
    RandomCuboid and sampler see the same numbers: chosen attempt, kept boxes, crop, sampled rows and extents agree.
    The float64 transform equals numpy's float64 np.dot and scale bit for bit."""
    from coda_neurips2023_b200._lib import lib, ptr, stream_of
    from coda_neurips2023_b200.datasets.device_pipeline import _f, _i, _rot_matrices
    rng = np.random.default_rng(0)
    b, n, g, ncand, ns = 3, 9000, 12, 100, 4000
    pts32 = (rng.integers(-256, 257, size=(b, n, 6)) / 64.0).astype(np.float32)
    boxes32 = np.zeros((b, g, 8), np.float32)
    for i in range(b):
        boxes32[i, :, 0:3] = pts32[i, rng.integers(0, n, size=g), 0:3]
    boxes32[..., 3:6] = 0.25
    boxes32[:, 0, 0:3] = 100.0                # outside every cloud: a chosen crop must drop it
    nbox = torch.tensor([g, 5, 0], dtype=torch.int32).cuda()
    npts = torch.tensor([n, 7000, n], dtype=torch.int32).cuda()
    draws = draw_augmentation_sunrgbd(np.random.default_rng(1), b)
    cr, cu = torch.from_numpy(draws["crop_range"]).cuda(), torch.from_numpy(draws["center_u"]).cuda()
    seed = torch.from_numpy(draws["seed"].astype(np.int64)).to(torch.int32).cuda()
    L = lib()
    res = {}
    for dt, sfx in ((torch.float32, ""), (torch.float64, "_f64")):
        pts = torch.from_numpy(pts32).to(dt).cuda()
        bx = torch.from_numpy(boxes32).to(dt).cuda()
        st = stream_of(pts)
        ext = torch.empty((b, 6), dtype=dt).cuda()
        assert getattr(L, "coda_points_extent" + sfx)(_i(b), _i(n), _i(6), ptr(npts), ptr(pts), ptr(ext), st) == 0
        rxyz = (ext[:, 3:] - ext[:, :3]).contiguous()
        scratch = torch.empty((b, ncand, 8), dtype=dt).cuda()
        chosen = torch.empty((b,), dtype=torch.int32).cuda()
        crop = torch.empty((b, 6), dtype=torch.float64).cuda()
        keep = torch.empty((b, g), dtype=torch.uint8).cuda()
        assert getattr(L, "coda_random_cuboid" + sfx)(_i(b), _i(n), _i(6), _i(ncand), _i(g), _i(8), _i(2000), _f(0.75),
                                                      ptr(npts), ptr(pts), ptr(rxyz), ptr(cr), ptr(cu), ptr(bx),
                                                      ptr(nbox), ptr(scratch), ptr(chosen), ptr(crop), ptr(keep),
                                                      st) == 0
        lst = torch.empty((b, n), dtype=torch.int32).cuda()
        cnt = torch.empty((b,), dtype=torch.int32).cuda()
        out = torch.empty((b, ns, 6), dtype=dt).cuda()
        ch = torch.empty((b, ns), dtype=torch.int32).cuda()
        dims = torch.empty((b, 6), dtype=dt).cuda()
        assert getattr(L, "coda_sample_points" + sfx)(_i(b), _i(n), _i(6), _i(ns), ptr(npts), ptr(pts), ptr(crop),
                                                      ptr(seed), ptr(lst), ptr(cnt), ptr(out), ptr(ch), ptr(dims),
                                                      st) == 0
        torch.cuda.synchronize()
        res[dt] = dict(ext=ext.double(), chosen=chosen, crop=crop, keep=keep, cnt=cnt, choice=ch, out=out.double(),
                       dims=dims.double())
    for k in res[torch.float32]:
        assert torch.equal(res[torch.float32][k], res[torch.float64][k]), k
    cropped = (res[torch.float64]["chosen"] >= 0) & (nbox > 0)
    assert cropped.any() and (res[torch.float64]["keep"][cropped, 0] == 0).all()
    # the float64 transform against numpy
    raw = rng.standard_normal((b, n, 6)) * 3
    flip = np.array([-1, 1, -1], np.float32)
    rot = _rot_matrices(draws["rot_angle"])
    pts = torch.from_numpy(raw).cuda()
    assert L.coda_points_flip2_rotate_scale_f64(
        _i(b), _i(n), _i(6), None, ptr(torch.from_numpy(flip).cuda()), ptr(torch.ones(b).cuda()),
        ptr(torch.from_numpy(rot).cuda()), ptr(torch.from_numpy(draws["scale"]).cuda()), ptr(pts), stream_of(pts)) == 0
    for i in range(b):
        e = raw[i].copy()
        e[:, 0] = flip[i] * e[:, 0]
        e[:, 0:3] = np.dot(e[:, 0:3], rot[i].T)
        e[:, 0:3] *= np.tile(draws["scale"][i], 3)[None]
        assert np.array_equal(pts[i].cpu().numpy(), e)
