"""torch restatement of the GIoU kernel's arithmetic (CHECKER for csrc/detr_kernels.cu
giou3d_kernel); follows reference utils/box_util.py:655-757.  The polygon clip runs in
oracle/box_oracle.c when built (fp32), else in the Python restatement below."""
import ctypes
import subprocess
from pathlib import Path

import numpy as np
import torch

_HERE = Path(__file__).resolve().parent
_BOX = None


def _box_lib():
    global _BOX
    if _BOX is None:
        so = _HERE / "liboracle_box.so"
        if not so.exists() or so.stat().st_mtime < (_HERE / "box_oracle.c").stat().st_mtime:
            subprocess.run(["make", "-C", str(_HERE)], check=True, capture_output=True)
        _BOX = ctypes.CDLL(str(so))
    return _BOX


def rotated_inter_areas(r1, r2, non_rot, nums_k2, k2_limit):
    r1 = np.ascontiguousarray(r1.numpy(), np.float32)
    r2 = np.ascontiguousarray(r2.numpy(), np.float32)
    nr = np.ascontiguousarray(non_rot.numpy(), np.float32)
    nk = np.ascontiguousarray(np.asarray(nums_k2), np.int32)
    out = np.zeros_like(nr)
    vp = ctypes.c_void_p
    _box_lib().oracle_rotated_inter_areas(r1.shape[0], r1.shape[1], r2.shape[1], int(k2_limit),
                                          r1.ctypes.data_as(vp), r2.ctypes.data_as(vp), nr.ctypes.data_as(vp),
                                          nk.ctypes.data_as(vp), out.ctypes.data_as(vp))
    return torch.from_numpy(out)


def _inside(cp1, cp2, p):
    return (cp2[0] - cp1[0]) * (p[1] - cp1[1]) > (cp2[1] - cp1[1]) * (p[0] - cp1[0])


def _intersect(cp1, cp2, s, e):
    f = np.float32
    dc = (f(cp1[0] - cp2[0]), f(cp1[1] - cp2[1]))
    dp = (f(s[0] - e[0]), f(s[1] - e[1]))
    n1 = f(cp1[0] * cp2[1]) - f(cp1[1] * cp2[0])
    n2 = f(s[0] * e[1]) - f(s[1] * e[0])
    n3 = f(1.0) / (f(dc[0] * dp[1]) - f(dc[1] * dp[0]))
    return (f((n1 * dp[0] - n2 * dc[0]) * n3), f((n1 * dp[1] - n2 * dc[1]) * n3))


def _clip_area(subj, clip):
    # like the kernel (csrc/box_geometry.cuh), on the eight points taken relative to clip[0]
    org = tuple(np.float32(v) for v in clip[0])
    out = [tuple(np.float32(v) - o for v, o in zip(p, org)) for p in subj]
    clip = [tuple(np.float32(v) - o for v, o in zip(p, org)) for p in clip]
    cp1 = clip[-1]
    for cp2 in clip:
        inp, out = out, []
        s = inp[-1]
        for e in inp:
            if _inside(cp1, cp2, e):
                if not _inside(cp1, cp2, s):
                    out.append(_intersect(cp1, cp2, s, e))
                out.append(e)
            elif _inside(cp1, cp2, s):
                out.append(_intersect(cp1, cp2, s, e))
            s = e
        cp1 = cp2
        if not out:
            return 0.0
    xs = np.array([p[0] for p in out], np.float32)
    ys = np.array([p[1] for p in out], np.float32)
    return float(abs(np.dot(xs, np.roll(ys, 1)) - np.dot(ys, np.roll(xs, 1))) * 0.5)


def giou3d_ref(c1, c2, nums_k2, rotated, rot_k2_limit=None):
    c1, c2 = c1.detach().float().cpu(), c2.detach().float().cpu()
    B, K1, K2 = c1.shape[0], c1.shape[1], c2.shape[1]
    lim = K2 if rot_k2_limit is None else rot_k2_limit
    eps = 1e-8
    ymax = torch.min(c1[:, :, 0, 1][:, :, None], c2[:, :, 0, 1][:, None, :])
    ymin = torch.max(c1[:, :, 4, 1][:, :, None], c2[:, :, 4, 1][:, None, :])
    height = (ymax - ymin).clamp(min=0)
    r1 = c1[:, :, [3, 2, 1, 0]][..., [0, 2]]
    r2 = c2[:, :, [3, 2, 1, 0]][..., [0, 2]]
    lt = torch.max(r1[:, :, 1][:, :, None, :], r2[:, :, 1][:, None, :, :])
    rb = torch.min(r1[:, :, 3][:, :, None, :], r2[:, :, 3][:, None, :, :])
    wh = (rb - lt).clamp(min=0)
    non_rot = wh[..., 0] * wh[..., 1]
    both = torch.cat((c1[:, :, None].expand(-1, -1, K2, -1, -1), c2[:, None].expand(-1, K1, -1, -1, -1)), dim=3)
    dx = both[..., 0].amax(-1) - both[..., 0].amin(-1)
    dy = both[..., 1].amax(-1) - both[..., 1].amin(-1)
    dz = both[..., 2].amax(-1) - both[..., 2].amin(-1)
    enclosing = dx.abs() * dy.abs() * dz.abs()

    def vol(c):
        def e(i, j):
            return torch.sqrt((c[:, :, i] - c[:, :, j]).pow(2).sum(-1).clamp(min=1e-6))
        return (e(0, 1) * e(1, 2) * e(0, 4)).clamp(min=eps)

    sum_vols = vol(c1)[:, :, None] + vol(c2)[:, None, :]
    good = (enclosing > 2 * eps) & (sum_vols > 4 * eps)
    inter = non_rot.clone()
    nk = [int(v) for v in nums_k2]
    if rotated:
        inter = rotated_inter_areas(r1, r2, non_rot, nk, lim)
    inter_vol = inter * height
    union = (sum_vols - inter_vol).clamp(min=eps)
    g = (inter_vol / union - (1 - union / enclosing)) * good
    mask = torch.zeros_like(g)
    for b in range(B):
        mask[b, :, : nk[b]] = 1
    return g * mask
