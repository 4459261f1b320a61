"""An fp64 twin of the pre-encoder's inference kernel (csrc/sa_infer_sm90.cu) built from the kernel's own operands,
and the fp64 module path it stands for.  CPU-importable: the GPU tests run the same code on CUDA tensors.

The kernel computes, per seed (64 neighbour rows):
    h1 = relu(A1(W1 x))                 fp32 FMAs, then split into 3 bf16 planes a0 + a1 + a2
    z2 = sum over 6 plane products      W2 on its 3 planes b0 + b1 + b2
    h2 = relu(A2(z2))                   fp32, split into 3 planes
    z3 = sum over 5 plane products      W3 on planes 0 and 1 ONLY (W3' = b0 + b1)
    out = relu(max over rows of A3(z3))
with A_l(v) = v * scale_l + shift_l the folded running-statistics BatchNorm (sa_mlp._folded_affine).

The twin forms the same plane products in fp64, each one separately, so that the twin without any one product can be
formed (test_sa_infer_twin_cpu checks that every product is visible above the bar).  What is left between the kernel
and the twin is fp32 rounding: of h1 and h2 before they are split (each to half an fp32 ulp), of the tensor-core
accumulators, and of the affine FMAs.

Layer 1 is restated exactly (the same fp32 FMAs in the same order), so h1 is the kernel's h1.

Conditioning.  For output element (seed, j), with the worst of the seed's 64 rows:
    cond_j = |scale3_j| * sum_k |H2_k * W3'_jk| + |shift3_j|,   H2_k = max(|h2_k|, |scale2_k z2_k| if h2_k > 0)
Every rounding the kernel makes downstream of h2 is a relative error of at most a few fp32 ulps (2^-24) on a term of
that sum or on the affine: the accumulators add 5 x 128 products (exact in fp32: bf16 x bf16) in k-steps of 16, and
each addition rounds to 2^-24 of the partial sum, which is at most the sum of magnitudes.  A rounding of h2_k by
2^-24 relative moves the sum by |W3'_jk h2_k| 2^-24, inside the same bound.  Layer-2 rounding reaches h2 through
z2's accumulator, at 2^-24 of |z2| scaled by scale2: where the affine cancels (running_var ~ 0 makes scale2 ~ 220 and
shift2 ~ -220 running_mean) that is far more than 2^-24 |h2|, hence H2 (a channel the ReLU zeroes passes no rounding
on).  The max and the ReLU are 1-Lipschitz.  A worst-case
sum of 640 roundings would be 2^-14.6 cond; rounding errors of independent signs add like a random walk, ~25 x 2^-24
= 2^-19.4 cond at the very worst element; the measured worst on random inputs is 0.32 x 2^-20 cond (every seed of
the evaluation shape included; DESIGN.md section 2, a5).  TWIN_BAR = 2^-20 sits between: 3x above what is measured,
and below the smallest plane product, so that removing any one of them is caught (the bar-power test measures each).

Against the exact module path (fp32 W3) the kernel also carries W3's 2-plane truncation, |W3 - W3'| <= 2^-16 |W3|
per weight, which moves the sum by at most 2^-16 cond: MODULE_BAR = 2^-16 + TWIN_BAR.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

GROUP = 64
WIDTHS = (64, 128, 256)
# (A plane, B plane) per product, in the kernel's order (operand_split.cuh prod_a / prod_b; sa_infer_sm90.cu l3_a /
# l3_b): smallest terms first
L2_PRODUCTS = ((1, 1), (2, 0), (0, 2), (1, 0), (0, 1), (0, 0))
L3_PRODUCTS = ((1, 1), (2, 0), (1, 0), (0, 1), (0, 0))
W3_PLANES = 2
TWIN_BAR = 2.0 ** -20
MODULE_BAR = 2.0 ** -16 + TWIN_BAR


def product_name(a: int, b: int) -> str:
    return f"a{a}b{b}"


# ---------------------------------------------------------------------- the bf16 operand split
def bf16_rn(x: np.ndarray) -> np.ndarray:
    """fp32 -> the nearest bf16 value (ties to even), as fp32: the rounding of __floats2bfloat162_rn for finite x"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def split_planes_np(x: np.ndarray, n: int) -> list[np.ndarray]:
    """next_plane (operand_split.cuh) restated: plane p is the bf16 rounding of what the planes before it left over;
    the subtraction is exact in fp32"""
    r = np.asarray(x, dtype=np.float32)
    planes = []
    for _ in range(n):
        p = bf16_rn(r)
        planes.append(p)
        r = (r - p).astype(np.float32)
    return planes


def split_planes(x: torch.Tensor, n: int = 3) -> list[torch.Tensor]:
    """the same split of an fp32 tensor on its own device (torch's fp32 -> bf16 cast rounds to nearest even)"""
    r = x.float()
    planes = []
    for _ in range(n):
        p = r.to(torch.bfloat16).float()
        planes.append(p)
        r = r - p
    return planes


# ---------------------------------------------------------------------- the kernel's operands
def folded_affine(blocks) -> torch.Tensor:
    from coda_neurips2023_b200 import sa_mlp

    return sa_mlp._folded_affine(blocks)


def blocks_of(mlp):
    """(conv, bn) pairs of a SharedMLP"""
    return [(blk.conv, blk.bn.bn) for blk in mlp]


def weight_planes_np(w: torch.Tensor) -> torch.Tensor:
    """(3, rows, k) planes of an fp32 weight by the numpy split (the CPU stand-in for ops._packed_weight)"""
    m = w.detach().reshape(w.shape[0], -1).float().cpu().numpy()
    return torch.from_numpy(np.stack(split_planes_np(m, 3))).to(w.device)


def weight_planes_packed(w: torch.Tensor) -> torch.Tensor:
    """(3, rows, k) planes the kernel reads: ops._packed_weight with the 3 planes shared_mlp_max_infer asks for"""
    from coda_neurips2023_b200 import ops

    wp = ops._packed_weight(w.reshape(w.shape[0], -1), False, 3)
    return wp[:, 0].float()


def weight_planes_exact(w: torch.Tensor) -> torch.Tensor:
    """(3, rows, k): the exact fp32 weight as plane 0, zero planes 1 and 2 (no split, no truncation)"""
    m = w.detach().reshape(w.shape[0], -1).float()
    return torch.cat([m[None], torch.zeros((2, *m.shape), dtype=m.dtype, device=m.device)])


def operands(blocks, packed: bool = True):
    """(w1, affine, w2 planes, w3 planes) of an eval-mode SharedMLP's (conv, bn) blocks, as the kernel reads them"""
    planes = weight_planes_packed if packed else weight_planes_np
    w1 = blocks[0][0].weight.detach().reshape(WIDTHS[0], -1).float()
    return w1, folded_affine(blocks).float(), planes(blocks[1][0].weight), planes(blocks[2][0].weight)


# ---------------------------------------------------------------------- the twin
def _rows(x: torch.Tensor) -> torch.Tensor:
    """(B, C0, npoint, 64) -> (B * npoint, 64, C0)"""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[3], x.shape[1])


def _affine(affine: torch.Tensor):
    a = affine.double()
    c1, c2, c3 = WIDTHS
    o = np.cumsum([0, c1, c1, c2, c2, c3, c3])
    return [a[o[i]:o[i + 1]] for i in range(6)]


def _fma32(a, b, c):
    """fmaf: the exact a * b + c (fp64 holds the product of two fp32 values exactly) rounded once to fp32"""
    return (a.double() * b.double() + c.double()).float()


def twin(x, w1, affine, w2p, w3p, drop=None, exact=False, want_cond=True):
    """x (B, C0, npoint, 64) -> (out (B * npoint, 256), cond (B * npoint, 256) or None), fp64, on x's device.

    w2p, w3p: weight planes (planes, rows, k) as fp32 values; W3 is read from its first W3_PLANES planes.
    drop: ("l2" | "l3", product index) leaves that plane product out.
    exact: activations stay fp64 and are carried as one plane (no fp32 rounding, no split) -- with the weights given
    as one exact plane this is the module path, which is how test_sa_infer_twin_cpu checks the twin's structure."""
    s1, h1s, s2, h2s, s3, h3s = _affine(affine)
    xr = _rows(x).double()
    dev = xr.device
    w2p, w3p = w2p.to(dev).double(), w3p.to(dev).double()

    def act_planes(v):
        if exact:
            return [v, torch.zeros_like(v), torch.zeros_like(v)]
        return [p.double() for p in split_planes(v.float(), 3)]

    def products(a_planes, b_planes, plist, layer):
        acc = None
        for i, (pa, pb) in enumerate(plist):
            if drop == (layer, i):
                continue
            t = a_planes[pa] @ b_planes[pb].t()
            acc = t if acc is None else acc + t
        return acc

    if exact:
        h1 = torch.relu((xr @ w1.to(dev).double().t()) * s1 + h1s)
    else:
        # layer 1 as the kernel runs it: fp32 FMAs over the channels in order, then the affine as one more FMA
        w1f, v = w1.to(dev).float(), torch.zeros((*xr.shape[:2], WIDTHS[0]), dtype=torch.float32, device=dev)
        for c in range(xr.shape[2]):
            v = _fma32(xr[..., c:c + 1], w1f[:, c], v)
        h1 = torch.relu(_fma32(v, s1, h1s)).double()
    z2 = products(act_planes(h1), w2p, L2_PRODUCTS, "l2")
    h2 = torch.relu(z2 * s2 + h2s)
    a3 = act_planes(h2)
    w3 = w3p[:W3_PLANES]
    z3 = products(a3, w3, L3_PRODUCTS, "l3")
    out = torch.relu((z3 * s3 + h3s).amax(dim=1))
    cond = None
    if want_cond:
        h2v = h2 if exact else h2.float().double()                  # the fp32 value the kernel splits
        # where the layer-2 affine cancels (|h2| << |scale2 z2|), h2 carries the rounding of z2 at z2's magnitude
        carried = torch.maximum(h2v.abs(), torch.where(h2v > 0, (z2 * s2).abs(), 0.0))
        mag = carried @ w3.sum(0).abs().t()
        cond = (s3.abs() * mag + h3s.abs()).amax(dim=1)
    return out, cond


def twin_chunked(x, w1, affine, w2p, w3p, scenes_per_chunk=1):
    """twin() over the scenes of x a few at a time (the evaluation shape does not fit at once)"""
    outs, conds = [], []
    for b0 in range(0, x.shape[0], scenes_per_chunk):
        o, c = twin(x[b0:b0 + scenes_per_chunk], w1, affine, w2p, w3p)
        outs.append(o)
        conds.append(c)
    return torch.cat(outs), torch.cat(conds)


def module_path(blocks, x):
    """fp64 module path of (conv, bn) blocks: Conv2d 1x1 -> eval-mode BatchNorm2d -> ReLU, three times, then
    F.max_pool2d over the neighbours -> (B * npoint, 256)"""
    with torch.no_grad():
        y = x.double()
        for conv, bn in blocks:
            y = F.conv2d(y, conv.weight.double())
            y = F.batch_norm(y, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(),
                             bn.bias.double(), False, 0.0, bn.eps)
            y = torch.relu(y)
        pooled = F.max_pool2d(y, kernel_size=[1, y.size(3)]).squeeze(-1)      # (B, 256, npoint)
    return pooled.permute(0, 2, 1).reshape(-1, pooled.shape[1])


# ---------------------------------------------------------------------- the cases the GPU tests use
def make_mlp(c0: int, seed: int):
    """the pre-encoder's MLP in eval mode (CPU) with non-trivial running statistics and some negative gamma"""
    from coda_neurips2023_b200.pointnet2 import pytorch_utils as pt_utils

    torch.manual_seed(seed)
    mlp = pt_utils.SharedMLP([c0, *WIDTHS], bn=True).eval()
    for m in mlp.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(-1.5, 1.5)
            m.bias.data.uniform_(-0.3, 0.3)
            m.running_mean.uniform_(-0.5, 0.5)
            m.running_var.uniform_(0.3, 3.0)
    for p in mlp.parameters():
        p.requires_grad_(False)
    return mlp


def make_input(b: int, c0: int, npoint: int, seed: int, scale: float = 1.0) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn((b, c0, npoint, GROUP), generator=g) * scale
