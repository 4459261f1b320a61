"""Shared by the golden generator (tests/golden/make_baseline_eval_golden.py) and the CPU / GPU tests of the 3DETR +
CLIP baseline head's test-time classification: the case's arguments and inputs, and OUR model built for it with the
weights, running statistics and small CLIP the generator gives the reference."""
import os
import warnings
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import torch

import model_parity_common as mpc
from coda_neurips2023_b200 import clip as clip_mod
from coda_neurips2023_b200 import synthetic
from coda_neurips2023_b200.models import build_model
from param_fill import fill_by_name
from running_stats_fill import fill_running_stats_by_name

GOLDEN = mpc.GOLDEN
STATS_SEED = 7
BATCH, NPOINTS = 3, 3000
NO_VIEW_SCENE = 2          # this scene's camera looks away from the room: no box has a usable crop
ZERO_QUERIES = (3, 17, 40)  # queries whose predicted size is forced to zero (skipped by the size test)
SCANNET_CALIB = GOLDEN / "baseline_eval_scannet"
IMAGE_HW = {"sunrgbd_image": (531, 730), "scannet50_image": (968, 1296)}


def golden_path(dataset_name):
    short = "scannet" if "scannet" in dataset_name else "sunrgbd"
    return GOLDEN / f"model_baseline_clip_eval_{short}.npz"

# the test_release_models.sh baseline arguments, at the small model size of the parity goldens
_BASE = dict(mpc._SMALL, model_name="3detrmulticlasshead", nqueries=128, train_range_max=10, test_range_max=46,
             if_clip_more_prompts=True)
DATASET_ARGS = {
    "sunrgbd_image": dict(dataset_name="sunrgbd_image"),
    "scannet50_image": dict(dataset_name="scannet50_image", train_range_max=10, test_range_max=60,
                            reset_scannet_num=50),
}


def args_for(dataset_name):
    return synthetic.make_args(**dict(_BASE, **DATASET_ARGS[dataset_name]))


def reference_args(dataset_name):
    import make_model_golden as mmg

    a = mmg.reference_args(dict(_BASE, **DATASET_ARGS[dataset_name]))
    a.if_only_novel_prompt = False
    a.if_with_clip = True
    return a


def make_inputs(dataset_name="sunrgbd_image") -> dict:
    """The test batch (numpy), in which NO_VIEW_SCENE's camera looks away from the room.  SUN RGB-D: that camera is
    turned half a turn about its x axis.  ScanNet: the synthetic poses look at the room of a training batch, whose
    flips and rotation the test path does not undo, so here it is the other scenes' cameras that are turned half a
    turn, towards the room.  A ScanNet batch still carries the camera as K / Rtilt here: the generator writes them
    to the calibration files, and neither run sees them in the batch."""
    if "scannet" in dataset_name:
        d = synthetic.make_batch(BATCH, NPOINTS, seed=5, image_hw=IMAGE_HW[dataset_name], camera="scannet")
        for b in range(BATCH):
            if b != NO_VIEW_SCENE:
                d["Rtilt"][b][:3, :3] = d["Rtilt"][b][:3, :3] @ np.diag([1.0, -1.0, -1.0])
    else:
        d = synthetic.make_batch(BATCH, NPOINTS, seed=5, image_hw=IMAGE_HW[dataset_name])
        d["Rtilt"][NO_VIEW_SCENE] = np.diag([1.0, -1.0, -1.0])
    return d


def scannet_calib_dir(b: int) -> Path:
    return SCANNET_CALIB / f"scene{b:04d}_00"


def squence_name(b: int) -> str:
    return str(10 * b + 3)


def scannet_names() -> dict:
    """calib_name / squence_name of a ScanNet test batch, pointing at the golden's calibration files."""
    return {"calib_name": [str(scannet_calib_dir(b)) for b in range(BATCH)],
            "squence_name": [squence_name(b) for b in range(BATCH)]}


def zero_sizes(box_processor) -> None:
    """Forces the predicted size of ZERO_QUERIES to zero in every scene and decoder layer."""
    size = box_processor.compute_predicted_size

    def sized(size_normalized, point_cloud_dims):
        s = size(size_normalized, point_cloud_dims).clone()
        s[:, list(ZERO_QUERIES)] = 0
        return s

    box_processor.compute_predicted_size = sized


@contextmanager
def class_lists():
    """Runs with the working directory where datasets/ holds the class lists (from tests/golden/), as a CoDA
    checkout has them."""
    import tempfile

    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.mkdir(Path(tmp) / "datasets")
        for name in ("all_classes_trainval_v1.npy", "scannet_200_classname_no_wall_floor.npy",
                     "scannet_200_class2id.npy"):
            os.symlink(GOLDEN / name, Path(tmp) / "datasets" / name)
        os.chdir(tmp)
        try:
            yield
        finally:
            os.chdir(cwd)


def build_ours(device, dataset_name="sunrgbd_image"):
    """OUR baseline head with the golden's weights (fill_by_name seed 3, running statistics seed 7, the small CLIP
    filled with seed 11) and text features, in eval mode on `device`."""
    args = args_for(dataset_name)
    cfg = synthetic.SyntheticDatasetConfig(args)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    tiny = clip_mod.CLIP(**mpc.TINY_CLIP).float().eval()
    fill_by_name(tiny, seed=11)
    for p in tiny.parameters():
        p.requires_grad = False
    model.clip_model = tiny
    model.clip_resolution = 224
    fill_by_name(model, seed=3)
    fill_running_stats_by_name(model, seed=STATS_SEED)
    golden = np.load(golden_path(dataset_name))
    model.text_features_fg_norm = torch.from_numpy(golden["text_features_fg_norm"])
    model.logit_scale = torch.tensor(float(golden["logit_scale"]))   # exp() of the CLIP the constructor saw
    zero_sizes(model.box_processor)
    model.to_device(device)
    model.eval()
    return model, golden


def test_batch(device, dataset_name="sunrgbd_image") -> dict:
    """The batch the golden's reference run saw: a ScanNet batch without K / Rtilt, naming its calibration files."""
    inputs = synthetic.to_device(make_inputs(dataset_name), device)
    if "scannet" in dataset_name:
        del inputs["K"], inputs["Rtilt"]
        inputs.update(scannet_names())
    return inputs


def run_ours(device, dataset_name="sunrgbd_image"):
    model, golden = build_ours(device, dataset_name)
    inputs = test_batch(device, dataset_name)
    with torch.no_grad():
        out = model(inputs, if_real_test=True)
    return model, out["outputs"], golden


def scannet_extent_cpu(corners_xyz, size_unnorm, inputs):
    """CPU restatement of coda_boxes_in_image with the ScanNet camera (include/coda_detr.h), in fp64 torch ops:
    corners (augmentation undone) -> inv(pose) -> K[:3, :3] -> per-corner clamp to [0, w - 1] x [0, h - 1] plus the
    offsets (image flip 1 = none) -> (int boxes, usable, fp64 extent)."""
    b = corners_xyz.shape[0]
    dd = torch.double
    pts = corners_xyz.to(dd) * inputs["scale_array"].to(dd).reshape(b, 1, 1, 3)
    pts = torch.matmul(pts, inputs["rot_array"].to(dd).reshape(b, 1, 3, 3))
    if "zx_flip_array" in inputs:
        pts = pts * torch.stack((torch.ones(b, dtype=dd), inputs["zx_flip_array"].to(dd).reshape(b),
                                 torch.ones(b, dtype=dd)), -1).reshape(b, 1, 1, 3)
    fx = inputs["flip_array"].to(dd).reshape(b, 1, 1)
    pts = torch.cat((pts[..., :1] * fx.unsqueeze(-1), pts[..., 1:]), -1)
    pose_inv = torch.linalg.inv(inputs["Rtilt"].to(dd)).reshape(b, 1, 4, 4)
    cam = torch.matmul(pts, pose_inv[..., :3, :3].transpose(-1, -2)) + pose_inv[..., :3, 3].unsqueeze(-2)
    uvw = torch.matmul(cam, inputs["K"].to(dd)[:, :3, :3].reshape(b, 1, 3, 3).transpose(-1, -2))
    d = uvw[..., 2]
    u, v = uvw[..., 0] / (d + 1e-32), uvw[..., 1] / (d + 1e-32)
    wmax = (inputs["ori_width"].to(dd) - 1).reshape(b, 1, 1)
    hmax = (inputs["ori_height"].to(dd) - 1).reshape(b, 1, 1)
    zero = torch.zeros((), dtype=dd)
    u = torch.minimum(torch.maximum(u, zero), wmax) + inputs["y_offset"].to(dd).reshape(b, 1, 1)
    v = torch.minimum(torch.maximum(v, zero), hmax) + inputs["x_offset"].to(dd).reshape(b, 1, 1)
    fl = inputs["image_flip_array"].to(dd).reshape(b, 1, 1)
    flen = inputs["flip_length"].to(dd).reshape(b, 1, 1)
    u = u * fl + (1 - fl) * (flen - 1 - u)
    ext = torch.stack((u.amin(-1), v.amin(-1), u.amax(-1), v.amax(-1)), -1)
    boxes = ext.to(torch.int32)
    usable = ((boxes[..., 2] - boxes[..., 0]) > 0) & ((boxes[..., 3] - boxes[..., 1]) > 0) & (d.amin(-1) >= 0) & \
        ~(size_unnorm.amax(-1) < 1e-16)
    return boxes, usable, ext


