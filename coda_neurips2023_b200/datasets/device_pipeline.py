"""The per-scene numpy pipeline of the reference's dataset `__getitem__`
(datasets/sunrgbd_anonymous_aligned_image.py:618-795) for a whole BATCH of raw scenes that already live in HBM:
point-cloud / box augmentation (flip about YZ, rotation about the up axis, scale), RandomCuboid (utils/random_cuboid.py), random sampling to `num_points` (utils/pc_util.py:24-32), the image
augmentation (:624-655), and the label tensors the model and the criterion read.  The ScanNet item
(datasets/scannet_anonymous_aligned_image.py:373-702) orders its steps differently -- crop and sample the raw scene
first, transform the sampled rows last, with a second flip -- and has its own class below (DeviceScanNetAugmentor).
The whole collated SUN RGB-D item, on its float64 scene files and bit-equal to the reference's, is
DeviceSunrgbdAugmentor at the end of this module.

Why on the device: the reference runs this in DataLoader workers, one scene at a time, on the host; at 275 scenes/s
per GPU that is ~14 M points/s of numpy work per GPU plus an 11 MB host-to-device copy per step.  Raw scenes are a
few GB for SUN RGB-D (10 335 scenes x ~50 k points x 12 B): they fit in HBM many times over, so the epoch loop
becomes index selection + five kernel launches (include/coda_data.h), no workers, no copies.

Randomness stays with the caller, as small arrays (`draw_augmentation`): the same role np.random plays in the
reference, which makes the device path a deterministic function that oracle/data_ref.py restates on the CPU.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from .._lib import check, lib, ptr, stream_of

_i = lambda v: ctypes.c_int(int(v))  # noqa: E731
_f = lambda v: ctypes.c_float(float(v))  # noqa: E731


def draw_augmentation(rng: np.random.Generator, batch: int, ncand: int = 100, augment: bool = True,
                      min_crop: float = 0.75, max_crop: float = 1.0, image_augment: bool = True) -> dict:
    """One step's random numbers (host, numpy) -- what the reference draws inside __getitem__ / RandomCuboid:
    flip (:663), rotation angle in +-30 degrees (:672), scale 0.85-1.15 (:700), per attempt a crop range in
    [min_crop, max_crop]^3 and a centre point (random_cuboid.py:43-50), a sampling seed (pc_util.py:28), and for the
    image a flip, per-channel gain 0.8-1.2 and shift +-0.05, a jitter seed (:630-645)."""
    p = {}
    if augment:
        p["flip"] = np.where(rng.random(batch) > 0.5, -1.0, 1.0).astype(np.float32)
        p["rot_angle"] = (rng.random(batch) * np.pi / 3 - np.pi / 6)
        p["scale"] = (rng.random(batch) * 0.3 + 0.85).astype(np.float32)
    else:
        p["flip"] = np.ones(batch, np.float32)
        p["rot_angle"] = np.zeros(batch)
        p["scale"] = np.ones(batch, np.float32)
    p["crop_range"] = min_crop + rng.random((batch, ncand, 3)) * (max_crop - min_crop)
    p["center_u"] = rng.random((batch, ncand)).astype(np.float32)
    p["seed"] = rng.integers(0, 2 ** 32, size=batch, dtype=np.uint32)
    if image_augment:
        p["image_flip"] = (rng.random(batch) > 0.5).astype(np.uint8)
        p["image_gain"] = (1 + 0.4 * rng.random((batch, 3)) - 0.2).astype(np.float32)
        p["image_shift"] = (0.1 * rng.random((batch, 3)) - 0.05).astype(np.float32)
        p["image_seed"] = rng.integers(0, 2 ** 32, size=batch, dtype=np.uint32)
    return p


def rotz(t: np.ndarray) -> np.ndarray:
    """(B,) angles -> (B, 3, 3) rotation about the up axis (utils/pc_util.py:125-129)"""
    c, s = np.cos(t), np.sin(t)
    z, o = np.zeros_like(c), np.ones_like(c)
    return np.stack((np.stack((c, -s, z), -1), np.stack((s, c, z), -1), np.stack((z, z, o), -1)), -2)


class DeviceSceneAugmentor:
    """raw scenes on the device -> the collated training batch.

    raw_points (B, Nmax, stride) fp32 with npts (B,) valid rows (xyz [+ colour]); raw_boxes (B, Gmax, 8) fp32 rows
    [cx, cy, cz, l/2, w/2, h/2, heading, class] in the upright depth frame with nbox (B,) valid rows
    (datasets/...:441-442 `_bbox.npy`)."""

    def __init__(self, num_points: int = 20000, max_num_obj: int = 64, num_angle_bin: int = 12, augment: bool = True,
                 use_random_cuboid: bool = True, random_cuboid_min_points: int = 30000, aspect: float = 0.75,
                 ncand: int = 100):
        self.num_points, self.max_num_obj, self.num_angle_bin = num_points, max_num_obj, num_angle_bin
        self.augment, self.use_random_cuboid = augment, use_random_cuboid
        self.min_points, self.aspect, self.ncand = random_cuboid_min_points, aspect, ncand

    # ------------------------------------------------------------------ kernels
    @torch.no_grad()
    def points(self, raw_points: torch.Tensor, npts: torch.Tensor, raw_boxes: torch.Tensor, nbox: torch.Tensor,
               params: dict):
        """-> dict(point_clouds (B, num_points, stride), choice, dims (B, 6), boxes (B, Gmax, 8) transformed,
        box_keep (B, Gmax) bool, chosen (B,) int32)"""
        if not raw_points.is_cuda:
            raise RuntimeError("DeviceSceneAugmentor: CPU not supported (tests/scannet_item_ref.py is the CPU restatement)")
        dev = raw_points.device
        b, nmax, stride = raw_points.shape
        gmax = raw_boxes.shape[1]
        pts = raw_points.detach().float().clone().contiguous()       # transformed in place
        npts_i = npts.to(device=dev, dtype=torch.int32).contiguous()
        nbox_i = nbox.to(device=dev, dtype=torch.int32).contiguous()
        up = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).to(dev)  # noqa: E731
        flip, scale = up(params["flip"], torch.float32), up(params["scale"], torch.float32)
        rot64 = rotz(np.asarray(params["rot_angle"], np.float64))
        rot = up(rot64.astype(np.float32), torch.float32)
        L = lib()
        st = stream_of(pts)
        with torch.cuda.device(dev):
            check(L.coda_scene_transform(_i(b), _i(nmax), _i(stride), ptr(npts_i), ptr(flip), ptr(rot), ptr(scale),
                                         ptr(pts), st), "scene_transform")
            # boxes: a handful of rows per scene (datasets/...:664-666, 675-677, 701-703), same float32 arithmetic
            boxes = raw_boxes.detach().float().clone()
            f, s = flip.view(b, 1), scale.view(b, 1)
            ang = up(np.asarray(params["rot_angle"], np.float64).astype(np.float32), torch.float32).view(b, 1)
            boxes[..., 0] = boxes[..., 0] * f
            boxes[..., 6] = torch.where(f < 0, math.pi - boxes[..., 6], boxes[..., 6]) - ang
            ctr = boxes[..., 0:3]
            boxes[..., 0:3] = torch.stack([(ctr[..., 0] * rot[:, j, 0:1] + ctr[..., 1] * rot[:, j, 1:2])
                                           + ctr[..., 2] * rot[:, j, 2:3] for j in range(3)], dim=-1) * s.unsqueeze(-1)
            boxes[..., 3:6] = boxes[..., 3:6] * s.unsqueeze(-1)
            boxes = boxes.contiguous()
            extent = torch.empty((b, 6), dtype=torch.float32, device=dev)
            check(L.coda_points_extent(_i(b), _i(nmax), _i(stride), ptr(npts_i), ptr(pts), ptr(extent), st),
                  "points_extent")
            range_xyz = (extent[:, 3:] - extent[:, :3]).contiguous()
            crop = torch.empty((b, 6), dtype=torch.float64, device=dev)
            chosen = torch.full((b,), -1, dtype=torch.int32, device=dev)
            keep = torch.ones((b, max(gmax, 1)), dtype=torch.uint8, device=dev)
            if self.augment and self.use_random_cuboid:
                cr = up(params["crop_range"], torch.float64)
                cu = up(params["center_u"], torch.float32)
                ncand = cr.shape[1]
                scratch = torch.empty((b, ncand, 8), dtype=torch.float32, device=dev)
                check(L.coda_random_cuboid(_i(b), _i(nmax), _i(stride), _i(ncand), _i(gmax), _i(boxes.shape[2]),
                                           _i(self.min_points), _f(self.aspect), ptr(npts_i), ptr(pts), ptr(range_xyz),
                                           ptr(cr), ptr(cu), ptr(boxes), ptr(nbox_i), ptr(scratch), ptr(chosen),
                                           ptr(crop), ptr(keep), st), "random_cuboid")
            else:
                crop[:, :3] = float("-inf")
                crop[:, 3:] = float("inf")
                keep = (torch.arange(max(gmax, 1), device=dev).view(1, -1) < nbox_i.view(b, 1)).to(torch.uint8)
            seed = up(np.asarray(params["seed"]).astype(np.int64), torch.int64).to(torch.int32).contiguous()   # bit pattern
            lst = torch.empty((b, nmax), dtype=torch.int32, device=dev)
            count = torch.empty((b,), dtype=torch.int32, device=dev)
            out = torch.empty((b, self.num_points, stride), dtype=torch.float32, device=dev)
            choice = torch.empty((b, self.num_points), dtype=torch.int32, device=dev)
            dims = torch.empty((b, 6), dtype=torch.float32, device=dev)
            check(L.coda_sample_points(_i(b), _i(nmax), _i(stride), _i(self.num_points), ptr(npts_i), ptr(pts), ptr(crop),
                                       ptr(seed), ptr(lst), ptr(count), ptr(out), ptr(choice), ptr(dims), st),
                  "sample_points")
        return dict(point_clouds=out, choice=choice, dims=dims, boxes=boxes, box_keep=keep[:, :gmax].bool(),
                    chosen=chosen, count=count, crop=crop, rot=rot64)

    @torch.no_grad()
    def images(self, images: torch.Tensor, params: dict) -> torch.Tensor:
        """(B, H, W, 3) uint8 -> augmented uint8 (datasets/...:624-655)"""
        if not images.is_cuda or images.dtype != torch.uint8:
            raise RuntimeError("images must be uint8 CUDA tensors (B, H, W, 3)")
        img = images.contiguous()
        b, h, w, _ = img.shape
        dev = img.device
        up = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).to(dev)  # noqa: E731
        flip = up(params["image_flip"], torch.uint8)
        gain, shift = up(params["image_gain"], torch.float32), up(params["image_shift"], torch.float32)
        seed = up(np.asarray(params["image_seed"]).astype(np.int64), torch.int64).to(torch.int32).contiguous()
        out = torch.empty_like(img)
        with torch.cuda.device(dev):
            check(lib().coda_image_augment(_i(b), _i(h), _i(w), ptr(img), ptr(flip), ptr(gain), ptr(shift), ptr(seed),
                                           ptr(out), stream_of(img)), "image_augment")
        return out

    # ------------------------------------------------------------------ labels (tiny tensors: plain tensor ops)
    @torch.no_grad()
    def labels(self, boxes: torch.Tensor, box_keep: torch.Tensor, dims: torch.Tensor, dataset_config) -> dict:
        """The ground-truth tensors of datasets/...:707-795 from the augmented boxes: kept boxes are packed to the
        front (RandomCuboid drops the others), padded to max_num_obj."""
        b, gmax, _ = boxes.shape
        g = self.max_num_obj
        dev = boxes.device
        order = torch.argsort((~box_keep).to(torch.int8), dim=1, stable=True)           # kept boxes first, in order
        bx = torch.gather(boxes.double(), 1, order.unsqueeze(-1).expand(-1, -1, boxes.shape[2]))
        present = torch.gather(box_keep, 1, order)
        pad = g - gmax
        if pad > 0:
            bx = torch.cat((bx, bx.new_zeros(b, pad, bx.shape[2])), 1)
            present = torch.cat((present, present.new_zeros(b, pad)), 1)
        bx, present = bx[:, :g], present[:, :g]
        mask = present.double()
        bx = bx * mask.unsqueeze(-1)
        two_pi = 2 * math.pi
        per = two_pi / self.num_angle_bin
        ang = bx[..., 6] % two_pi
        shifted = (ang + per / 2) % two_pi
        cls = torch.floor(shifted / per).long()
        res = shifted - (cls.double() * per + per / 2)
        raw_sizes = bx[..., 3:6] * 2
        # re-encoded angle, as class2angle_batch does (:771-773): centre of the bin + residual, wrapped to (-pi, pi]
        raw_angles = cls.double() * per + res
        raw_angles = torch.where(raw_angles > math.pi, raw_angles - two_pi, raw_angles)
        # axis-aligned extent of the heading-rotated box (:722-741)
        c, s = torch.cos(-bx[..., 6]), torch.sin(-bx[..., 6])
        l, w, h = bx[..., 3], bx[..., 4], bx[..., 5]
        ex = (c * l).abs() + (s * w).abs()
        ey = (s * l).abs() + (c * w).abs()
        centers = bx[..., 0:3]
        dmin, dmax = dims[:, :3].double().unsqueeze(1), dims[:, 3:].double().unsqueeze(1)
        span = dmax - dmin
        out = {
            "gt_box_present": mask.float(),
            "gt_box_centers": centers.float(),
            "gt_box_centers_normalized": (((centers - dmin) / span) * mask.unsqueeze(-1)).float(),
            "gt_box_sizes": raw_sizes.float(),
            "gt_box_sizes_normalized": (raw_sizes / span).float(),
            "gt_box_angles": (raw_angles * mask).float(),
            "gt_angle_class_label": cls * present.long(),
            "gt_angle_residual_label": (res * mask).float(),
            "gt_box_extent": torch.stack((2 * ex, 2 * ey, 2 * h), -1).float(),
            "gt_box_sem_cls_label": bx[..., 7].long() * present.long(),
            "point_cloud_dims_min": dims[:, :3].contiguous(),
            "point_cloud_dims_max": dims[:, 3:].contiguous(),
        }
        if dataset_config is not None:
            out["gt_box_corners"] = dataset_config.box_parametrization_to_corners(
                centers.float(), raw_sizes.float(), raw_angles.float()) * mask.float().view(b, g, 1, 1)
        return out


# ---------------------------------------------------------------------------------------------------- ScanNet
# The ScanNet item (datasets/scannet_anonymous_aligned_image.py:373-702) is a different pipeline from SUN RGB-D's:
# RandomCuboid runs on the RAW scene, sampling to num_points follows, and the flips (about YZ and about XZ), the
# rotation and the scale run last, on the sampled rows, in float64 against the float32 cloud.  The image is placed on
# a white image_size canvas before it is augmented.  tests/scannet_item_ref.py restates it on the CPU.

def draw_augmentation_scannet(rng: np.random.Generator, batch: int, ncand: int = 100, min_crop: float = 0.5,
                              max_crop: float = 1.0) -> dict:
    """One batch's random numbers for the ScanNet item, in the roles np.random plays there: image flip, per-channel
    gain 0.8-1.2 and shift +-0.05, jitter seed (:458-491); per RandomCuboid attempt a crop range and a centre draw
    (random_cuboid.py:43-50); the sampling seed (pc_util.py:28); flip about YZ, flip about XZ, rotation in +-30
    degrees, scale 0.85-1.15 (:545-604).  The `*_u` entries are the uniforms the derived values come from, with the
    reference's formulas (rot_angle = u * pi / 3 - pi / 6, scale = u * 0.3 + 0.85) in float64."""
    p = {"image_flip": (rng.random(batch) > 0.5).astype(np.uint8)}
    p["image_gain_u"], p["image_shift_u"] = rng.random((batch, 3)), rng.random((batch, 3))
    p["image_gain"] = (1 + 0.4 * p["image_gain_u"] - 0.2).astype(np.float32)
    p["image_shift"] = (0.1 * p["image_shift_u"] - 0.05).astype(np.float32)
    p["image_seed"] = rng.integers(0, 2 ** 32, size=batch, dtype=np.uint32)
    p["crop_range"] = min_crop + rng.random((batch, ncand, 3)) * (max_crop - min_crop)
    p["center_u"] = rng.random((batch, ncand)).astype(np.float32)
    p["seed"] = rng.integers(0, 2 ** 32, size=batch, dtype=np.uint32)
    p["flip_yz"] = np.where(rng.random(batch) > 0.5, -1.0, 1.0).astype(np.float32)
    p["flip_xz"] = np.where(rng.random(batch) > 0.5, -1.0, 1.0).astype(np.float32)
    p["rot_u"], p["scale_u"] = rng.random(batch), rng.random(batch)
    p["rot_angle"] = p["rot_u"] * np.pi / 3 - np.pi / 6
    p["scale"] = p["scale_u"] * 0.3 + 0.85
    return p


def identity_draws_scannet(p: dict) -> dict:
    """the same draws without the point-cloud flips, rotation and scale (crop, sampling and image unchanged)"""
    q = dict(p)
    b = len(p["seed"])
    q["flip_yz"], q["flip_xz"] = np.ones(b, np.float32), np.ones(b, np.float32)
    q["rot_u"], q["scale_u"] = np.full(b, 0.5), np.full(b, 0.5)
    q["rot_angle"], q["scale"] = np.zeros(b), np.ones(b)
    return q


def _rot_matrices(rot_angle) -> np.ndarray:
    """(B, 3, 3) float64 pc_util.rotz of each angle, entry for entry as the reference builds it"""
    out = []
    for t in np.asarray(rot_angle, np.float64).reshape(-1):
        c, s = np.cos(float(t)), np.sin(float(t))
        out.append(np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]))
    return np.stack(out)


@torch.no_grad()
def augment_frames(frames, image_size, params: dict):
    """frames (B, h, w, 3) uint8 RGB (or a list of per-scene frames) -> (augmented (B, H, W, 3) uint8 canvas,
    x_offset (B,), y_offset (B,), ori_width, ori_height): each frame on a white image_size = (W, H) canvas at
    ((H - h) // 2, (W - w) // 2), then coda_image_augment of the canvas, border included.  The ScanNet and SUN RGB-D
    items pad and augment their frames the same way (scannet_anonymous_aligned_image.py:385-398, :458-491;
    sunrgbd_anonymous_aligned_image.py:397-410, :624-655)."""
    W, H = image_size
    frames = list(frames)
    b = len(frames)
    if any((not f.is_cuda) or f.dtype != torch.uint8 or f.dim() != 3 or f.shape[2] != 3 for f in frames):
        raise RuntimeError("frames must be uint8 CUDA tensors (h, w, 3), RGB")
    if any(f.shape[0] > H or f.shape[1] > W for f in frames):
        raise ValueError(f"a frame is larger than the {W} x {H} canvas")
    dev = frames[0].device
    canvas = torch.full((b, H, W, 3), 255, dtype=torch.uint8, device=dev)
    xo, yo = [], []
    for i, f in enumerate(frames):
        h, w = int(f.shape[0]), int(f.shape[1])
        xo.append((H - h) // 2)
        yo.append((W - w) // 2)
        canvas[i, xo[-1]:xo[-1] + h, yo[-1]:yo[-1] + w] = f
    up = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).to(dev)  # noqa: E731
    flip = up(params["image_flip"], torch.uint8)
    gain, shift = up(params["image_gain"], torch.float32), up(params["image_shift"], torch.float32)
    seed = up(np.asarray(params["image_seed"]).astype(np.int64), torch.int64).to(torch.int32).contiguous()
    out = torch.empty_like(canvas)
    with torch.cuda.device(dev):
        check(lib().coda_image_augment(_i(b), _i(H), _i(W), ptr(canvas), ptr(flip), ptr(gain), ptr(shift),
                                       ptr(seed), ptr(out), stream_of(canvas)), "image_augment")
    i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=dev)  # noqa: E731
    return (out, i64(xo), i64(yo), i64([int(f.shape[1]) for f in frames]), i64([int(f.shape[0]) for f in frames]))


def _rotate(cor, R, ctr):
    """cor (.., 8, 3) @ R^T + ctr, float64, written out (3 x 3: no GEMM library call)"""
    return torch.stack([cor[..., 0] * R[..., k, 0:1] + cor[..., 1] * R[..., k, 1:2] + cor[..., 2] * R[..., k, 2:3]
                        for k in range(3)], -1) + ctr.unsqueeze(-2)


def _corners_camera(centers, sizes, angles):
    """box_parametrization_to_corners_np: camera-frame corners of roty(angle) boxes (utils/box_util.py:297-327)"""
    c2 = centers[..., [0, 2, 1]].clone()
    c2[..., 1] *= -1
    c, s = torch.cos(angles).double(), torch.sin(angles).double()
    z, o = torch.zeros_like(c), torch.ones_like(c)
    R = torch.stack((torch.stack((c, z, s), -1), torch.stack((z, o, z), -1), torch.stack((-s, z, c), -1)), -2)
    l, w, h = (sizes[..., k:k + 1] / 2 for k in range(3))
    cor = torch.stack((torch.cat((l, l, -l, -l, l, l, -l, -l), -1), torch.cat((h, h, h, h, -h, -h, -h, -h), -1),
                       torch.cat((w, -w, -w, w, w, -w, -w, w), -1)), -1).double()
    return _rotate(cor, R, c2.double()).float()


def _corners_xyz(centers, sizes, angles):
    """depth-frame corners of rotz(angle) boxes: get_3d_box_batch_np_xyz (utils/box_util.py:360-381) of -angle"""
    c, s = torch.cos(angles).double(), torch.sin(angles).double()
    z, o = torch.zeros_like(c), torch.ones_like(c)
    R = torch.stack((torch.stack((c, -s, z), -1), torch.stack((s, c, z), -1), torch.stack((z, z, o), -1)), -2)
    l, w, h = (sizes[..., k:k + 1] / 2 for k in range(3))
    cor = torch.stack((torch.cat((-l, l, l, -l, -l, l, l, -l), -1), torch.cat((w, w, -w, -w, w, w, -w, -w), -1),
                       torch.cat((h, h, h, h, -h, -h, -h, -h), -1)), -1).double()
    return _rotate(cor, R, centers.double()).float()


class DeviceScanNetAugmentor:
    """raw ScanNet scenes on the device -> the collated training batch of the reference's ScanNet item.

    raw_points (B, Nmax, 6) fp32 `_pc.npy` rows [x, y, z, r, g, b] with npts (B,) valid; bbox_rows (B, Gmax, 8) fp32
    `_bbox.npy` rows [cx, cy, cz, dx/2, dy/2, dz/2, heading, class id] with nbox (B,) valid; frames (B, h, w, 3) uint8
    RGB (or a list of per-scene (h, w, 3) frames).  `select_range` is the class-id list the split keeps
    (train_range_list for training); the kept boxes' class becomes 0 (one class-agnostic label)."""

    def __init__(self, select_range, num_points: int = 40000, max_num_obj: int = 64, num_angle_bin: int = 12,
                 random_cuboid_min_points: int = 30000, aspect: float = 0.8, image_size=(1296, 968),
                 use_color: bool = False, use_height: bool = False):
        for flag, on in (("use_color", use_color), ("use_height", use_height)):
            if on:
                raise NotImplementedError(f"DeviceScanNetAugmentor does not implement --{flag}")
        self.select_range = [int(c) for c in select_range]
        self.num_points, self.max_num_obj, self.num_angle_bin = num_points, max_num_obj, num_angle_bin
        self.min_points, self.aspect = random_cuboid_min_points, aspect
        self.image_size = tuple(int(v) for v in image_size)       # (W, H)

    # ------------------------------------------------------------------ kernels
    @torch.no_grad()
    def select_boxes(self, bbox_rows: torch.Tensor, nbox: torch.Tensor):
        """rows of the selected classes packed to the front, class column 0 (:433-438) -> (rows, count int32)"""
        b, gmax, _ = bbox_rows.shape
        dev = bbox_rows.device
        valid = torch.arange(gmax, device=dev).view(1, -1) < nbox.to(dev).view(b, 1)
        sel = valid & torch.isin(bbox_rows[..., 7], torch.tensor(self.select_range, dtype=bbox_rows.dtype, device=dev))
        order = torch.argsort((~sel).to(torch.int8), dim=1, stable=True)
        rows = torch.gather(bbox_rows.float(), 1, order.unsqueeze(-1).expand(-1, -1, 8))
        cnt = sel.sum(1).to(torch.int32)
        rows = rows * (torch.arange(gmax, device=dev).view(1, -1, 1) < cnt.view(b, 1, 1))
        rows[..., 7] = 0
        worst = int(cnt.max()) if b else 0
        if worst > self.max_num_obj:
            raise ValueError(f"a scene has {worst} boxes of the selected classes; max_num_obj is {self.max_num_obj}")
        return rows.contiguous(), cnt.contiguous()

    @torch.no_grad()
    def points(self, raw_points: torch.Tensor, npts: torch.Tensor, boxes: torch.Tensor, nbox: torch.Tensor,
               params: dict) -> dict:
        """RandomCuboid on the raw scenes, sampling, then flips / rotation / scale of the sampled rows (:493-606).
        boxes (B, G, 8) are select_boxes' rows.  -> point_clouds (B, N, 3), point_clouds_rgb (B, N, 6), pcl_color,
        dims (B, 6) of the transformed cloud, chosen (B,), box_keep (B, G), list_pos / choice (B, N), rot (B, 3, 3)"""
        if not raw_points.is_cuda:
            raise RuntimeError("DeviceScanNetAugmentor: CPU not supported (tests/scannet_item_ref.py is the CPU restatement)")
        dev = raw_points.device
        b, nmax, stride = raw_points.shape
        if stride != 6:
            raise ValueError(f"raw_points must be (B, Nmax, 6) rows [x, y, z, r, g, b]; got stride {stride}")
        gmax, n = boxes.shape[1], self.num_points
        pts = raw_points.detach().float().contiguous()
        npts_i = npts.to(device=dev, dtype=torch.int32).contiguous()
        nbox_i = nbox.to(device=dev, dtype=torch.int32).contiguous()
        up = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).to(dev)  # noqa: E731
        L = lib()
        st = stream_of(pts)
        with torch.cuda.device(dev):
            extent = torch.empty((b, 6), dtype=torch.float32, device=dev)
            check(L.coda_points_extent(_i(b), _i(nmax), _i(stride), ptr(npts_i), ptr(pts), ptr(extent), st),
                  "points_extent")
            range_xyz = (extent[:, 3:] - extent[:, :3]).contiguous()
            cr, cu = up(params["crop_range"], torch.float64), up(params["center_u"], torch.float32)
            ncand = cr.shape[1]
            scratch = torch.empty((b, ncand, 8), dtype=torch.float32, device=dev)
            chosen = torch.empty((b,), dtype=torch.int32, device=dev)
            crop = torch.empty((b, 6), dtype=torch.float64, device=dev)
            keep = torch.ones((b, max(gmax, 1)), dtype=torch.uint8, device=dev)
            bx = boxes.float().contiguous()
            check(L.coda_random_cuboid(_i(b), _i(nmax), _i(stride), _i(ncand), _i(gmax), _i(8), _i(self.min_points),
                                       _f(self.aspect), ptr(npts_i), ptr(pts), ptr(range_xyz), ptr(cr), ptr(cu),
                                       ptr(bx), ptr(nbox_i), ptr(scratch), ptr(chosen), ptr(crop), ptr(keep), st),
                  "random_cuboid")
            seed = up(np.asarray(params["seed"]).astype(np.int64), torch.int64).to(torch.int32).contiguous()
            lst = torch.empty((b, nmax), dtype=torch.int32, device=dev)
            count = torch.empty((b,), dtype=torch.int32, device=dev)
            out = torch.empty((b, n, stride), dtype=torch.float32, device=dev)
            rgb = torch.empty((b, n, 6), dtype=torch.float32, device=dev)
            choice = torch.empty((b, n), dtype=torch.int32, device=dev)
            list_pos = torch.empty((b, n), dtype=torch.int32, device=dev)
            dims = torch.empty((b, 6), dtype=torch.float32, device=dev)
            check(L.coda_sample_points_ex(_i(b), _i(nmax), _i(stride), _i(n), _i(6), ptr(npts_i), ptr(pts), ptr(crop),
                                          ptr(seed), ptr(lst), ptr(count), ptr(out), ptr(choice), ptr(list_pos),
                                          ptr(rgb), ptr(dims), st), "sample_points_ex")
            pc = out[..., 0:3].contiguous()
            fyz, fxz = up(params["flip_yz"], torch.float32), up(params["flip_xz"], torch.float32)
            rot64 = _rot_matrices(params["rot_angle"])
            rot, scale = up(rot64, torch.float64), up(params["scale"], torch.float64)
            for t, w in ((pc, 3), (rgb, 6)):
                check(L.coda_points_flip2_rotate_scale(_i(b), _i(n), _i(w), None, ptr(fyz), ptr(fxz), ptr(rot),
                                                       ptr(scale), ptr(t), st), "points_flip2_rotate_scale")
            check(L.coda_points_extent(_i(b), _i(n), _i(3), None, ptr(pc), ptr(dims), st), "points_extent")
        return dict(point_clouds=pc, point_clouds_rgb=rgb, pcl_color=rgb[..., 3:6].contiguous(), dims=dims,
                    chosen=chosen, box_keep=keep[:, :gmax].bool(), list_pos=list_pos, choice=choice, count=count,
                    crop=crop, rot=rot64)

    @torch.no_grad()
    def images(self, frames, params: dict):
        """frames -> (augmented (B, H, W, 3) uint8 canvas, x_offset (B,), y_offset (B,), ori_width, ori_height):
        augment_frames on the image_size canvas (:385-398, :458-491)"""
        return augment_frames(frames, self.image_size, params)

    # ------------------------------------------------------------------ labels (64 boxes a scene: tensor ops)
    @torch.no_grad()
    def labels(self, boxes: torch.Tensor, box_keep: torch.Tensor, dims: torch.Tensor, params: dict) -> dict:
        """The ground-truth tensors of :530-700 from select_boxes' rows and RandomCuboid's box_keep, with the
        reference's float32 statements (the heading in float32, the centres through the points' transform)."""
        b, gmax, _ = boxes.shape
        g, dev = self.max_num_obj, boxes.device
        order = torch.argsort((~box_keep).to(torch.int8), dim=1, stable=True)
        kept = torch.gather(boxes.float(), 1, order.unsqueeze(-1).expand(-1, -1, boxes.shape[2]))[..., 0:7]
        present = torch.gather(box_keep, 1, order)
        tb = torch.zeros((b, g, 7), dtype=torch.float32, device=dev)
        mask = torch.zeros((b, g), dtype=torch.float32, device=dev)
        k = min(g, gmax)
        tb[:, :k] = kept[:, :k] * present[:, :k, None]
        mask[:, :k] = present[:, :k].float()
        up = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).to(dev)  # noqa: E731
        fyz, fxz = up(params["flip_yz"], torch.float32), up(params["flip_xz"], torch.float32)
        rot, scale = up(_rot_matrices(params["rot_angle"]), torch.float64), up(params["scale"], torch.float64)
        pi32 = torch.tensor(np.float32(np.pi), device=dev)
        head = tb[..., 6]
        head = torch.where(fyz.view(b, 1) < 0, pi32 - head, head)
        head = torch.where(fxz.view(b, 1) < 0, pi32 - head, head)
        head = head - up(np.asarray(params["rot_angle"], np.float64).astype(np.float32), torch.float32).view(b, 1)
        # centres: the same flips, float64 rotation and float64 scale as the points (:549-603)
        with torch.cuda.device(dev):
            check(lib().coda_points_flip2_rotate_scale(_i(b), _i(g), _i(7), None, ptr(fyz), ptr(fxz), ptr(rot),
                                                       ptr(scale), ptr(tb), stream_of(tb)), "points_flip2_rotate_scale")
        sizes = (tb[..., 3:6].double() * scale.view(b, 1, 1)).float()
        centers = tb[..., 0:3]
        raw_sizes = sizes * 2 * mask[..., None]
        raw_angles = head * -1 * mask
        # angle2class in float32 (a float32 angle against Python floats, :144-160)
        two_pi = torch.full_like(raw_angles, np.float32(2 * np.pi))
        per = 2 * np.pi / float(self.num_angle_bin)
        shifted = torch.remainder(torch.remainder(raw_angles, two_pi) + np.float32(per / 2), two_pi)
        cls = torch.trunc(shifted / torch.full_like(shifted, np.float32(per))).long()
        res = shifted - (cls.double() * per + per / 2).float()
        dmin, dmax = dims[:, None, :3], dims[:, None, 3:]
        span = dmax - dmin
        corners = _corners_camera(centers, raw_sizes, raw_angles)
        corners_xyz = _corners_xyz(centers, raw_sizes, raw_angles)
        return {
            "gt_box_corners": corners, "gt_box_corners_xyz": corners_xyz,
            "gt_box_centers": centers.contiguous(),
            "gt_box_centers_normalized": ((centers - dmin) / span) * mask[..., None],
            "gt_angle_class_label": cls * mask.long(),
            "gt_angle_residual_label": res * mask,
            "gt_box_sem_cls_label": torch.zeros((b, g), dtype=torch.int64, device=dev),
            "gt_box_present": mask,
            "gt_box_sizes": raw_sizes, "gt_box_sizes_normalized": raw_sizes * (1.0 / span),
            "gt_box_angles": raw_angles,
            "point_cloud_dims_min": dims[:, :3].contiguous(), "point_cloud_dims_max": dims[:, 3:].contiguous(),
        }

    # ------------------------------------------------------------------ the whole batch
    @torch.no_grad()
    def batch(self, raw_points, npts, bbox_rows, nbox, frames, K, Rtilt, params: dict) -> dict:
        """The reference's ScanNet items for B scenes after default collate: every key the model, the criterion and
        boxes_in_image(camera="scannet") read.  K / Rtilt (B, 4, 4) are the colour intrinsics and camera-to-world
        poses (models.model_3detr.ScanNetCalibration reads them)."""
        boxes, cnt = self.select_boxes(bbox_rows, nbox)
        pts = self.points(raw_points, npts, boxes, cnt, params)
        lab = self.labels(boxes, pts["box_keep"], pts["dims"], params)
        img, xo, yo, ow, oh = self.images(frames, params)
        dev = raw_points.device
        b = raw_points.shape[0]
        f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64).to(dev)  # noqa: E731
        rot = pts["rot"]
        out = dict(lab)
        out.update(point_clouds=pts["point_clouds"], point_clouds_rgb=pts["point_clouds_rgb"],
                   pcl_color=pts["pcl_color"], input_image=img, x_offset=xo, y_offset=yo, ori_width=ow,
                   ori_height=oh, K=f64(K), Rtilt=f64(Rtilt),
                   flip_array=f64(np.asarray(params["flip_yz"], np.float64).reshape(b, 1)),
                   zx_flip_array=f64(np.asarray(params["flip_xz"], np.float64).reshape(b, 1)),
                   rot_array=f64(np.stack([np.linalg.inv(np.transpose(r)) for r in rot])),
                   scale_array=f64((1.0 / np.tile(np.asarray(params["scale"], np.float64).reshape(b, 1), 3))
                                   .reshape(b, 1, 3)),
                   rot_angle=f64(np.asarray(params["rot_angle"], np.float64).reshape(b)),
                   image_flip_array=f64(np.where(np.asarray(params["image_flip"]) != 0, 0.0, 1.0).reshape(b, 1)),
                   flip_length=torch.full((b,), self.image_size[0], dtype=torch.int64, device=dev),
                   scan_idx=torch.arange(b, dtype=torch.int64, device=dev))
        return out


# ---------------------------------------------------------------------------------------------------- SUN RGB-D
# The SUN RGB-D item (datasets/sunrgbd_anonymous_aligned_image.py:383-900) flips, rotates and scales the WHOLE raw
# scene first, then crops it with RandomCuboid and samples it.  Its `_pc.npz` / `_bbox.npy` arrays are float64 (VoteNet's
# sunrgbd_data.py writes the depth points as scipy.io.loadmat returns MATLAB doubles), so every point and box step
# runs in float64 until the final float32 casts, and point_cloud_dims_min / max stay float64.  tests/sunrgbd_item_ref.py
# restates it on the CPU.

def draw_augmentation_sunrgbd(rng: np.random.Generator, batch: int, ncand: int = 100, min_crop: float = 0.75,
                              max_crop: float = 1.0) -> dict:
    """One batch's random numbers for the SUN RGB-D item, in the reference's call order: image flip, per-channel gain
    and shift uniforms, jitter seed (:630-649); point flip, rotation and scale uniforms (:665-704); per RandomCuboid
    attempt a crop-range and a centre uniform (random_cuboid.py:43-50); the sampling seed (pc_util.py:28).  The `*_u`
    entries are the uniforms numpy would return; the derived values use the reference's formulas in float64
    (rot_angle = u * pi / 3 - pi / 6, scale = u * 0.3 + 0.85, crop_range = min_crop + u * (max_crop - min_crop))."""
    p = {"image_flip": (rng.random(batch) > 0.5).astype(np.uint8)}
    p["image_gain_u"], p["image_shift_u"] = rng.random((batch, 3)), rng.random((batch, 3))
    p["image_gain"] = (1 + 0.4 * p["image_gain_u"] - 0.2).astype(np.float32)
    p["image_shift"] = (0.1 * p["image_shift_u"] - 0.05).astype(np.float32)
    p["image_seed"] = rng.integers(0, 2 ** 32, size=batch, dtype=np.uint32)
    p["flip"] = np.where(rng.random(batch) > 0.5, -1.0, 1.0).astype(np.float32)
    p["rot_u"], p["scale_u"] = rng.random(batch), rng.random(batch)
    p["rot_angle"] = (p["rot_u"] * np.pi / 3) - np.pi / 6
    p["scale"] = p["scale_u"] * 0.3 + 0.85
    p["crop_u"] = rng.random((batch, ncand, 3))
    p["crop_range"] = min_crop + p["crop_u"] * (max_crop - min_crop)
    p["center_u"] = rng.random((batch, ncand)).astype(np.float32)
    p["seed"] = rng.integers(0, 2 ** 32, size=batch, dtype=np.uint32)
    return p


def identity_draws_sunrgbd(p: dict) -> dict:
    """the same draws without the point-cloud flip, rotation and scale (crop, sampling and image unchanged)"""
    q = dict(p)
    b = len(p["seed"])
    q["flip"] = np.ones(b, np.float32)
    q["rot_u"], q["scale_u"] = np.full(b, 0.5), np.full(b, 0.5)
    q["rot_angle"], q["scale"] = np.zeros(b), np.ones(b)
    return q


def _box_rotations(boxes: torch.Tensor, cnt: torch.Tensor) -> torch.Tensor:
    """(B, G, 8) transformed float64 boxes -> (B, G, 3, 3) float64 pc_util.rotz(-1 * heading) of each valid row, on
    the host.  The entries are numpy's cos / sin of each float64 heading, evaluated one scalar at a time as
    my_compute_box_3d does (sunrgbd_anonymous_aligned_image.py:288-289): the device's double cos / sin are not
    correctly rounded and could differ from them in the last bit.  Rows past cnt stay zero."""
    heads = boxes[..., 6].cpu().numpy()
    counts = cnt.cpu().tolist()
    out = np.zeros(heads.shape + (3, 3))
    for i, n in enumerate(counts):
        for q in range(int(n)):
            t = -1 * heads[i, q]
            c, s = np.cos(t), np.sin(t)
            out[i, q] = ((c, -s, 0), (s, c, 0), (0, 0, 1))
    return torch.from_numpy(out).to(boxes.device)


class DeviceSunrgbdAugmentor:
    """raw SUN RGB-D scenes on the device -> the collated training batch of the reference's SUN RGB-D item.

    raw_points (B, N, 6) float64 `_pc.npz` rows [x, y, z, r, g, b], every scene with all N rows valid (the item
    returns the whole raw scene as point_clouds_rgb, and default collate needs one N); bbox_rows (B, Gmax, 8) float64
    `_bbox.npy` rows [cx, cy, cz, l/2, w/2, h/2, heading, class] with nbox (B,) valid; frames (B, h, w, 3) uint8 RGB
    (or a list of per-scene frames); K / Rtilt (B, 3, 3) as the calib text gives them (order='F').  Boxes of a class in
    [train_range_min, train_range_max) are kept, with class 0 and their own class as the seen class."""

    def __init__(self, train_range_min: int, train_range_max: int, nqueries: int, num_points: int = 20000,
                 max_num_obj: int = 64, num_angle_bin: int = 12, random_cuboid_min_points: int = 30000,
                 aspect: float = 0.75, image_size=(730, 531), use_color: bool = False, use_height: bool = False):
        for flag, on in (("use_color", use_color), ("use_height", use_height)):
            if on:
                raise NotImplementedError(f"DeviceSunrgbdAugmentor does not implement --{flag}")
        self.train_min, self.train_max, self.nqueries = int(train_range_min), int(train_range_max), int(nqueries)
        self.num_points, self.max_num_obj, self.num_angle_bin = num_points, max_num_obj, num_angle_bin
        self.min_points, self.aspect = random_cuboid_min_points, aspect
        self.image_size = tuple(int(v) for v in image_size)       # (W, H)

    # ------------------------------------------------------------------ kernels
    @torch.no_grad()
    def select_boxes(self, bbox_rows: torch.Tensor, nbox: torch.Tensor):
        """rows of a train class packed to the front, class column 0 (:476-499) -> (rows float64, seen class int64,
        count int32)"""
        b, gmax, _ = bbox_rows.shape
        dev = bbox_rows.device
        valid = torch.arange(gmax, device=dev).view(1, -1) < nbox.to(dev).view(b, 1)
        train = torch.arange(self.train_min, self.train_max, dtype=torch.float64, device=dev)
        sel = valid & torch.isin(bbox_rows[..., 7], train)
        order = torch.argsort((~sel).to(torch.int8), dim=1, stable=True)
        rows = torch.gather(bbox_rows, 1, order.unsqueeze(-1).expand(-1, -1, 8))
        cnt = sel.sum(1).to(torch.int32)
        rows = rows * (torch.arange(gmax, device=dev).view(1, -1, 1) < cnt.view(b, 1, 1))
        seen = rows[..., 7].to(torch.int64)
        rows[..., 7] = 0
        worst = int(cnt.max()) if b else 0
        if worst > self.max_num_obj:
            raise ValueError(f"a scene has {worst} boxes of a train class; max_num_obj is {self.max_num_obj}")
        return rows.contiguous(), seen, cnt.contiguous()

    @torch.no_grad()
    def points(self, raw_points: torch.Tensor, boxes: torch.Tensor, nbox: torch.Tensor, params: dict) -> dict:
        """Flip about YZ, rotation and scale of the whole scene and of select_boxes' rows, RandomCuboid, sampling
        (:660-771), all in float64.  -> point_clouds_rgb (B, N, 6) float64 (the transformed raw scene), sampled
        (B, num_points, 6) float64, dims (B, 6) float64, boxes (B, G, 8) transformed, box_keep (B, G), chosen, choice"""
        dev = raw_points.device
        b, n, stride = raw_points.shape
        gmax, ns = boxes.shape[1], self.num_points
        pts = raw_points.detach().clone().contiguous()                  # transformed in place: point_clouds_rgb
        bx = boxes.detach().clone().contiguous()
        npts_i = torch.full((b,), n, dtype=torch.int32, device=dev)
        nbox_i = nbox.to(device=dev, dtype=torch.int32).contiguous()
        up = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).to(dev)  # noqa: E731
        flip, ones = up(params["flip"], torch.float32), torch.ones((b,), dtype=torch.float32, device=dev)
        rot, scale = up(_rot_matrices(params["rot_angle"]), torch.float64), up(params["scale"], torch.float64)
        ang = up(np.asarray(params["rot_angle"], np.float64), torch.float64).view(b, 1)
        L = lib()
        st = stream_of(pts)
        with torch.cuda.device(dev):
            check(L.coda_points_flip2_rotate_scale_f64(_i(b), _i(n), _i(stride), None, ptr(flip), ptr(ones), ptr(rot),
                                                       ptr(scale), ptr(pts), st), "points_flip2_rotate_scale_f64")
            # boxes (:666-670, :678-680, :707-709): heading pi - h under the flip, then minus the angle; the centres
            # through the points' kernel; the half sizes times the float64 scale
            head = torch.where(flip.view(b, 1) < 0, math.pi - bx[..., 6], bx[..., 6])
            check(L.coda_points_flip2_rotate_scale_f64(_i(b), _i(gmax), _i(8), None, ptr(flip), ptr(ones), ptr(rot),
                                                       ptr(scale), ptr(bx), st), "points_flip2_rotate_scale_f64")
            bx[..., 6] = head - ang
            bx[..., 3:6] = bx[..., 3:6] * scale.view(b, 1, 1)
            extent = torch.empty((b, 6), dtype=torch.float64, device=dev)
            check(L.coda_points_extent_f64(_i(b), _i(n), _i(stride), None, ptr(pts), ptr(extent), st),
                  "points_extent_f64")
            range_xyz = (extent[:, 3:] - extent[:, :3]).contiguous()
            cr, cu = up(params["crop_range"], torch.float64), up(params["center_u"], torch.float32)
            ncand = cr.shape[1]
            scratch = torch.empty((b, ncand, 8), dtype=torch.float64, device=dev)
            chosen = torch.empty((b,), dtype=torch.int32, device=dev)
            crop = torch.empty((b, 6), dtype=torch.float64, device=dev)
            keep = torch.ones((b, max(gmax, 1)), dtype=torch.uint8, device=dev)
            check(L.coda_random_cuboid_f64(_i(b), _i(n), _i(stride), _i(ncand), _i(gmax), _i(8), _i(self.min_points),
                                           _f(self.aspect), ptr(npts_i), ptr(pts), ptr(range_xyz), ptr(cr), ptr(cu),
                                           ptr(bx), ptr(nbox_i), ptr(scratch), ptr(chosen), ptr(crop), ptr(keep), st),
                  "random_cuboid_f64")
            seed = up(np.asarray(params["seed"]).astype(np.int64), torch.int64).to(torch.int32).contiguous()
            lst = torch.empty((b, n), dtype=torch.int32, device=dev)
            count = torch.empty((b,), dtype=torch.int32, device=dev)
            out = torch.empty((b, ns, stride), dtype=torch.float64, device=dev)
            choice = torch.empty((b, ns), dtype=torch.int32, device=dev)
            dims = torch.empty((b, 6), dtype=torch.float64, device=dev)
            check(L.coda_sample_points_f64(_i(b), _i(n), _i(stride), _i(ns), ptr(npts_i), ptr(pts), ptr(crop),
                                           ptr(seed), ptr(lst), ptr(count), ptr(out), ptr(choice), ptr(dims), st),
                  "sample_points_f64")
        return dict(point_clouds_rgb=pts, sampled=out, dims=dims, boxes=bx, box_keep=keep[:, :gmax].bool(),
                    chosen=chosen, choice=choice, count=count, crop=crop)

    # ------------------------------------------------------------------ labels (64 boxes a scene: tensor ops)
    @torch.no_grad()
    def labels(self, boxes: torch.Tensor, seen: torch.Tensor, box_keep: torch.Tensor, dims: torch.Tensor,
               box_rot: torch.Tensor) -> dict:
        """The ground-truth tensors of :719-867 from the transformed float64 boxes, RandomCuboid's box_keep and
        box_rot (B, G, 3, 3) float64 = rotz(-heading) of every box (_box_rotations), all in select_boxes' order."""
        b, gmax, _ = boxes.shape
        g, dev = self.max_num_obj, boxes.device
        order = torch.argsort((~box_keep).to(torch.int8), dim=1, stable=True)
        k = min(g, gmax)
        kept = torch.zeros((b, g, 8), dtype=torch.float64, device=dev)
        present = torch.zeros((b, g), dtype=torch.bool, device=dev)
        seen_cls = torch.zeros((b, g), dtype=torch.int64, device=dev)
        kept[:, :k] = torch.gather(boxes, 1, order.unsqueeze(-1).expand(-1, -1, 8))[:, :k]
        present[:, :k] = torch.gather(box_keep, 1, order)[:, :k]
        seen_cls[:, :k] = torch.gather(seen, 1, order)[:, :k]
        R = torch.zeros((b, g, 3, 3), dtype=torch.float64, device=dev)
        R[:, :k] = torch.gather(box_rot, 1, order[..., None, None].expand(-1, -1, 3, 3))[:, :k]
        kept = kept * present[..., None]
        seen_cls = seen_cls * present
        mask = present.double()
        sizes = (kept[..., 3:6] * 2).float()
        # angle2class on the float64 heading (:144-160 of the config, Python float semantics)
        two_pi, per = 2 * math.pi, 2 * math.pi / float(self.num_angle_bin)
        shifted = torch.remainder(torch.remainder(kept[..., 6], two_pi) + per / 2, two_pi)
        cls = torch.trunc(shifted / per).long() * present.long()
        res = ((shifted - (cls.double() * per + per / 2)) * mask).float()
        # class2angle_batch (:255-263): float64 from the int class and the float32 residual
        angles = cls.double() * per + res.double()
        angles = torch.where(angles > math.pi, angles - two_pi, angles)
        angles32 = angles.float()
        # my_compute_box_3d (:288-298): np.dot(rotz(-heading), corners) through the fp64 kernel, one "scene" per box,
        # then the centre of the axis-aligned box around the corners
        l, w, h = (kept[..., k_:k_ + 1] for k_ in range(3, 6))
        cor = torch.stack((torch.cat((-l, l, l, -l, -l, l, l, -l), -1), torch.cat((w, w, -w, -w, w, w, -w, -w), -1),
                           torch.cat((h, h, h, h, -h, -h, -h, -h), -1)), -1).contiguous()
        R = R.contiguous()
        nb = b * g
        ones32 = torch.ones((nb,), dtype=torch.float32, device=dev)
        ones64 = torch.ones((nb,), dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            check(lib().coda_points_flip2_rotate_scale_f64(_i(nb), _i(8), _i(3), None, ptr(ones32), ptr(ones32),
                                                           ptr(R), ptr(ones64), ptr(cor), stream_of(cor)),
                  "points_flip2_rotate_scale_f64")
        cor = cor + kept[..., None, 0:3]
        centers = ((cor.amin(-2) + cor.amax(-2)) / 2 * mask[..., None]).float()
        dmin, dmax = dims[:, None, :3], dims[:, None, 3:]
        span = dmax - dmin
        valid = present & (seen_cls < self.train_max)
        image_label = torch.zeros((b, self.train_max + 1), dtype=torch.int64, device=dev)
        image_label.scatter_(1, torch.where(valid, seen_cls, self.train_max), 1)
        return {
            "gt_box_corners": _corners_camera(centers, sizes, angles32),
            "gt_box_corners_xyz": _corners_xyz(centers, sizes, -angles32),
            "gt_box_centers": centers,
            "gt_box_centers_normalized": ((((centers.double() - dmin) * 1.0) / span + 0.0) * mask[..., None]).float(),
            "gt_image_class_label": image_label[:, :self.train_max].contiguous(),
            "gt_box_sem_cls_label": torch.zeros((b, g), dtype=torch.int64, device=dev),
            "gt_box_seen_sem_cls_label": seen_cls,
            "gt_box_present": mask.float(),
            "gt_box_sizes": sizes,
            "gt_box_sizes_normalized": (sizes.double() * (1.0 / span)).float(),
            "gt_box_angles": angles32,
            "gt_angle_class_label": cls,
            "gt_angle_residual_label": res,
            "point_cloud_dims_min": dims[:, :3].contiguous(), "point_cloud_dims_max": dims[:, 3:].contiguous(),
        }

    # ------------------------------------------------------------------ the whole batch
    @torch.no_grad()
    def batch(self, raw_points, npts, bbox_rows, nbox, frames, K, Rtilt, draws: dict) -> dict:
        """The reference's SUN RGB-D items for B scenes after default collate: every key the item returns except the
        strings (calib_name, im_name) and uv_2d, which nothing on the training path reads.  npts (B,) must equal N
        for every scene."""
        if not torch.is_tensor(raw_points) or raw_points.dtype != torch.float64:
            raise TypeError("raw_points must be float64 (the _pc.npz arrays are float64; the item computes in float64)")
        if not raw_points.is_cuda:
            raise RuntimeError("DeviceSunrgbdAugmentor: CPU not supported (tests/sunrgbd_item_ref.py is the CPU "
                               "restatement)")
        b, n, stride = raw_points.shape
        if stride != 6:
            raise ValueError(f"raw_points must be (B, N, 6) rows [x, y, z, r, g, b]; got stride {stride}")
        counts = torch.as_tensor(npts).reshape(-1).tolist()
        if len(counts) != b or any(int(c) != n for c in counts):
            raise ValueError(f"every scene must have all N = {n} raw rows (point_clouds_rgb is the whole raw scene and "
                             f"default collate needs one N); got counts {counts}")
        if bbox_rows.dtype != torch.float64:
            raise TypeError("bbox_rows must be float64 (the _bbox.npy arrays are float64)")
        dev = raw_points.device
        boxes, seen, cnt = self.select_boxes(bbox_rows.to(dev), nbox)
        pts = self.points(raw_points, boxes, cnt, draws)
        out = self.labels(pts["boxes"], seen, pts["box_keep"], pts["dims"], _box_rotations(pts["boxes"], cnt))
        img, xo, yo, ow, oh = augment_frames(frames, self.image_size, draws)
        f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64).to(dev)  # noqa: E731
        rot = _rot_matrices(draws["rot_angle"])
        out.update(point_clouds=pts["sampled"][..., 0:3].float(), point_clouds_rgb=pts["point_clouds_rgb"].float(),
                   discovery_novel=torch.zeros((b, self.nqueries), dtype=torch.float64, device=dev),
                   scan_idx=torch.arange(b, dtype=torch.int64, device=dev),
                   K=f64(K).reshape(b, 3, 3), Rtilt=f64(Rtilt).reshape(b, 3, 3), input_image=img,
                   x_offset=xo, y_offset=yo, trans_mtx=torch.eye(2, dtype=torch.float64, device=dev).repeat(b, 1, 1),
                   ori_width=ow, ori_height=oh,
                   flip_array=f64(np.asarray(draws["flip"], np.float64).reshape(b, 1)),
                   scale_array=f64((1.0 / np.tile(np.asarray(draws["scale"], np.float64).reshape(b, 1), 3))
                                   .reshape(b, 1, 3)),
                   rot_array=f64(np.stack([np.linalg.inv(np.transpose(r)) for r in rot])),
                   image_flip_array=f64(np.where(np.asarray(draws["image_flip"]) != 0, 0.0, 1.0).reshape(b, 1)),
                   flip_length=torch.full((b,), self.image_size[0], dtype=torch.int64, device=dev))
        return out
