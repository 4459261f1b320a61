"""The CLIP crop kernel (coda_crop_resize_normalize_ex, csrc/image_kernels.cu) against fp64, pixel by pixel, at the
SUN RGB-D and ScanNet image sizes and at a small resolution, on boxes chosen for the kernel's edges: 1 x 1 boxes and
slivers, edges around the resolution, both centring parities, boxes on the right and bottom border, whole images,
the last image of the batch and given-up crops.  Then the bit relations between the kernel's forms (fp16 = fp32
rounded, every tile height, patch-major = NCHW unfolded, repeatability), guard words around the output, and the
limits (65535 crops, refusals).  tests/test_crop_discovery_paths_cpu.py maps the case lists below through the
kernel's path rules and checks that every tile height, hrow branch and scale regime is run.

The fp64 value v of a pixel is the separable sum with the per-axis weights of oracle/ref_crop.py (the fp32 weights of
ATen's antialiased bicubic).  The kernel sums the same weights in fp32, so its byte must be rint(clip(v, 0, 255))
wherever v is further than DELTA from a rounding boundary k + 1/2; nearer than that it may be one level off."""
import ctypes
import zlib

import numpy as np
import pytest
import torch

import crop_discovery_paths as P
import ref_crop
from coda_neurips2023_b200 import ops
from coda_neurips2023_b200._lib import lib

pytestmark = pytest.mark.gpu

SHAPES = {                             # name: (images, h, w, res)
    "sunrgbd": (8, 531, 730, 224),
    "scannet": (8, 968, 1296, 224),    # tile height 8, 25 taps: the tightest carve-up
    "small": (8, 120, 160, 36),        # a resolution that is not a multiple of the tile height
    "large": (2, 2000, 2000, 224),     # tile height 2, 37 taps
    "mid": (4, 170, 200, 160),         # tile_rows = 64 runs three tiles, the last one partial
}
TILE_ROWS = (1, 2, 4, 8, 16, 32, 64)
PATCHES = (16, 32)
MANY = (4, 64, 96, 16, 65535)          # images, h, w, res, crops: the most crops one launch takes
TOO_LARGE = ((1, 200, 2400, 224), (1, 16, 16, 2048))   # 45 taps; shared memory past the limit at one tile row

# fp32 accumulation bound of the kernel's separable sum, per unit of 255 * sum|wx| * sum|wy|: every tap of both
# passes is one fused multiply-add (at most 2^-23 relative with the product rounding of an unfused form), plus
# W_ULPS units of 2^-23 for the weights, whose cubic the compiler evaluates with fused multiply-adds where numpy
# rounds every step (a few ulps of the filter's unit sum)
EPS = 2.0 ** -23
W_ULPS = 4
MEAN64 = np.float32(ops.CLIP_MEAN).astype(np.float64)
STD64 = np.float32(ops.CLIP_STD).astype(np.float64)


def _images(name):
    """low-frequency content with sharp detail: random blocks upsampled, plus noise on one image in two"""
    nimg, h, w, _ = SHAPES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    base = torch.from_numpy(rng.integers(0, 256, (nimg, 3, max(h // 10, 2), max(w // 10, 2))).astype(np.float32))
    img = torch.nn.functional.interpolate(base, size=(h, w), mode="bilinear", align_corners=False)
    noise = torch.from_numpy(rng.normal(0, 40, (nimg, 3, h, w)).astype(np.float32))
    img = img + noise * (torch.arange(nimg) % 2).view(-1, 1, 1, 1)
    return img.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def crop_cases(name):
    """-> scene (n,) int32, boxes (n, 4) int32 [xmin, ymin, xmax, ymax], valid (n,) bool"""
    nimg, h, w, res = SHAPES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()) + 1)
    last = nimg - 1
    rows = []

    def add(s, x0, y0, x1, y1, v=True):
        assert 0 <= x0 < x1 <= w and 0 <= y0 < y1 <= h
        rows.append((s % nimg, x0, y0, x1, y1, v))

    add(0, 0, 0, w, h)                                   # the whole image: the longest filters
    add(last, 0, 0, w, h)                                # ... of the last image (scene offset)
    add(last, 0, 0, 1, 1)                                # 1 x 1 boxes
    add(1, w // 2, h // 3, w // 2 + 1, h // 3 + 1)
    add(1, 5, 0, 6, h)                                   # 1 x N and N x 1 slivers, on the bottom / right border
    add(2, 0, 7, w, 8)
    add(3, 10, 10, 11, 10 + min(res // 2, h - 10))
    add(4, 3, 20, 3 + min(res // 3, w - 3), 21)
    if name != "large":
        for e in (res - 1, res, res + 1):                # edge around the resolution, both centring parities
            for short in (e - 3, e - 4):
                add(5, 1, 2, 1 + e, 2 + short)
                add(last, w - short, h - e, w, h)        # the bottom-right corner
        add(6, w - 37, h - 50, w, h)
        add(6, w - 1, 0, w, 9)
        add(7 % nimg, 0, h - 1, 11, h)
        add(2, 10, 10, 100, 90, False)                   # given-up crops: exact zeros
        add(last, 0, 0, w, h, False)
        add(0, 0, 0, 1, 1, False)
        target = 60
    else:
        add(1, 100, 300, 1900, 1950)
        add(0, 0, 0, 1999, 1000, False)
        target = 12
    while len(rows) < target:
        x0, y0 = int(rng.integers(0, w - 1)), int(rng.integers(0, h - 1))
        x1, y1 = int(rng.integers(x0 + 1, w + 1)), int(rng.integers(y0 + 1, h + 1))
        add(int(rng.integers(0, nimg)), x0, y0, x1, y1, bool(rng.random() > 0.1))
    a = np.array(rows, dtype=np.int64)
    return a[:, 0].astype(np.int32), a[:, 1:5].astype(np.int32), a[:, 5].astype(bool)


def _weights64(edge, res):
    """(res, edge) fp64 matrix of ref_crop's fp32 weights, and per output index the tap count and sum|w|"""
    W = np.zeros((res, edge))
    for o, (lo, wt) in enumerate(ref_crop._weights(np.float32(edge) / np.float32(res), res, edge)):
        W[o, lo:lo + len(wt)] = wt
    return W, (W != 0).sum(1), np.abs(W).sum(1)


def _ref64(img, box, res):
    """fp64 pre-rounding values (3, res, res) of one crop and the per-pixel DELTA (res, res)"""
    wc, hc, edge, xb, yb = P.crop_geometry(box)
    x0, y0 = int(box[0]), int(box[1])
    canvas = torch.full((3, edge, edge), 255.0, dtype=torch.float64, device="cuda")
    canvas[:, yb:yb + hc, xb:xb + wc] = img[y0:y0 + hc, x0:x0 + wc].permute(2, 0, 1).double()
    W, n, s = _weights64(edge, res)
    Wd = torch.from_numpy(W).cuda()
    v = (Wd @ canvas @ Wd.T).cpu().numpy()           # fp64: the summation order is below 1e-12 of a level
    delta = 255.0 * np.outer(s, s) * EPS * (n[:, None] + n[None, :] + W_ULPS)
    return v, delta


def _levels(out):
    """the kernel's byte per pixel from its fp32 output, in fp64 (exact: the fp32 chain is far inside half a level)"""
    o = out.double().cpu().numpy()
    return np.rint((o * STD64[:, None, None] + MEAN64[:, None, None]) * 255.0)


def _normalised32(u8, steps=False):
    """the kernel's normalisation, (u8 / 255 - mean) / std, step by step in fp32 (with `steps`: the quotient, the
    difference and the result)"""
    u = u8.astype(np.float32)
    m, s = np.float32(ops.CLIP_MEAN)[:, None, None], np.float32(ops.CLIP_STD)[:, None, None]
    d = u / np.float32(255.0)
    t = d - m
    r = t / s
    return (d, t, r) if steps else r


def normalisation_error(o, u8):
    """-> (|o - fp64 value|, its bound, the same error in ulps of the fp64 value) for fp32 outputs o of levels u8.

    The fp32 chain rounds u / 255, then the difference, then the quotient, so its error is at most
    (ulp(u / 255) / 2 + ulp(u / 255 - mean) / 2) / std + ulp(result) / 2.  Near u / 255 = mean the difference
    cancels: the first term stays at the size of an ulp of u / 255 while the value shrinks, so the error is an
    absolute one of about 1e-7 and can reach far more than 2 ulps of the value (170 ulps for channel 2 at level 104,
    where the value is -1.3e-3).  No fp32 evaluation of this formula avoids that, so the bound is absolute."""
    ch = (slice(None), None, None)
    ref = (u8 / 255.0 - MEAN64[ch]) / STD64[ch]
    d, t, r = _normalised32(u8, steps=True)
    ulp = lambda x: np.spacing(np.abs(x)).astype(np.float64)  # noqa: E731
    bound = (ulp(d) + ulp(t)) / (2.0 * STD64[ch]) + ulp(r) / 2.0 + 1e-12
    err = np.abs(o.astype(np.float64) - ref)
    ulps = err / ulp(ref.astype(np.float32))
    return err, bound, ulps


def _check_against_fp64(out, imgs, scene, boxes, valid, res, stats):
    for i in range(len(boxes)):
        if not valid[i]:
            assert (out[i] == 0).all(), f"given-up crop {i} is not zero"
            continue
        v, delta = _ref64(imgs[int(scene[i])], boxes[i], res)
        u8 = _levels(out[i])
        exp = np.rint(np.clip(v, 0.0, 255.0))
        near = np.abs(v - (np.floor(v) + 0.5)) <= delta
        bad = (u8 != exp) & ~near
        assert not bad.any(), (f"crop {i} box {boxes[i].tolist()}: {int(bad.sum())} pixels off their fp64 level, "
                               f"first at {np.argwhere(bad)[0].tolist()}, v {v[bad][0]!r}, kernel {u8[bad][0]}")
        assert (np.abs(u8 - exp) <= 1).all(), f"crop {i}: a pixel near a rounding boundary more than 1 level off"
        o = out[i].cpu().numpy()
        assert np.array_equal(o, _normalised32(u8)), f"crop {i}: normalisation differs from its fp32 steps"
        err, bound, ulps = normalisation_error(o, u8)
        assert (err <= bound).all(), f"crop {i}: normalised value past the fp32 rounding bound"
        stats["err"] = max(stats.get("err", 0.0), float(err.max()))
        stats["ulps"] = max(stats.get("ulps", 0.0), float(ulps.max()))
        stats["near"] = stats.get("near", 0) + int(near.sum())
        stats["pixels"] = stats.get("pixels", 0) + near.size
        stats["delta"] = max(stats.get("delta", 0.0), float(delta.max()))


def _crop(imgs, scene, boxes, valid, res, **kw):
    return ops.crop_resize_normalize(imgs, torch.from_numpy(scene).cuda(), torch.from_numpy(boxes).cuda(),
                                     torch.from_numpy(valid).cuda(), res, **kw)


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


@pytest.mark.parametrize("name", list(SHAPES))
def test_crops_match_fp64_levels(name):
    """every pixel of every case against fp64; the fraction within DELTA of a rounding boundary is reported"""
    _, h, w, res = SHAPES[name]
    imgs = _images(name).cuda()
    scene, boxes, valid = crop_cases(name)
    out = _crop(imgs, scene, boxes, valid, res, dtype=torch.float32)
    stats = {}
    _check_against_fp64(out, imgs, scene, boxes, valid, res, stats)
    frac = stats["near"] / stats["pixels"]
    print(f"\n{name} ({h} x {w} -> {res}): {len(boxes)} crops, worst normalised error {stats['err']:.2e} "
          f"({stats['ulps']:.1f} ulp of the value), {100 * frac:.3f}% of pixels within delta "
          f"(max delta {stats['delta']:.2e})")
    assert frac < 0.01


@pytest.mark.parametrize("name", list(SHAPES))
def test_forms_are_bit_identical(name):
    """fp16 = fp32 rounded to half; every tile height; patch-major = NCHW unfolded; two runs agree"""
    _, _, _, res = SHAPES[name]
    imgs = _images(name).cuda()
    scene, boxes, valid = crop_cases(name)
    out = _crop(imgs, scene, boxes, valid, res, dtype=torch.float32)
    assert torch.equal(_crop(imgs, scene, boxes, valid, res, dtype=torch.float32), out), "two runs differ"
    half = _crop(imgs, scene, boxes, valid, res, dtype=torch.float16)
    assert torch.equal(half, out.half()), "fp16 output is not the fp32 output rounded"
    for tr in TILE_ROWS:
        assert torch.equal(_crop(imgs, scene, boxes, valid, res, dtype=torch.float32, tile_rows=tr), out), tr
    n = len(boxes)
    for p in (p for p in PATCHES if res % p == 0):
        g = res // p
        for dtype, ref in ((torch.float32, out), (torch.float16, half)):
            pm = _crop(imgs, scene, boxes, valid, res, dtype=dtype, patch=p)
            assert torch.equal(pm, ref.view(n, 3, g, p, g, p).permute(0, 2, 4, 1, 3, 5)), (p, dtype)


def test_scannet_crops_match_torchvision():
    """the reference's op sequence (crop, white canvas, torchvision Resize) at the ScanNet size: within one level,
    fewer than 1e-3 of the pixels flipped"""
    _, _, _, res = SHAPES["scannet"]
    imgs = _images("scannet").cuda()
    scene, boxes, valid = crop_cases("scannet")
    out = _crop(imgs, scene, boxes, valid, res, dtype=torch.float32)
    mean = torch.tensor(ops.CLIP_MEAN, device="cuda").view(3, 1, 1)
    std = torch.tensor(ops.CLIP_STD, device="cuda").view(3, 1, 1)
    for i in np.flatnonzero(valid):
        u8 = ref_crop.torchvision_sequence(imgs[int(scene[i])], [int(v) for v in boxes[i]], res)
        diff = (out[i] - (u8 / 255.0 - mean) / std).abs() * std * 255.0
        assert diff.max() <= 1.01, f"crop {i}: more than one level off torchvision"
        assert (diff > 0.5).float().mean() < 1e-3, f"crop {i}: too many rounding flips"


GUARD = 64
SENTINEL = {torch.float32: -7777.0, torch.float16: -777.0}


def _entry(imgs, scene, boxes, valid, res, ncrops, out_half, patch, work, out):
    """coda_crop_resize_normalize_ex itself, writing from out's first element -> its status"""
    nimg, h, w, _ = imgs.shape
    sc, bx = torch.from_numpy(scene).cuda(), torch.from_numpy(boxes).cuda()
    vd = torch.from_numpy(valid.astype(np.uint8)).cuda()
    m, s = (ctypes.c_float * 3)(*ops.CLIP_MEAN), (ctypes.c_float * 3)(*ops.CLIP_STD)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    i = ctypes.c_int
    return lib().coda_crop_resize_normalize_ex(i(nimg), i(h), i(w), i(ncrops), i(res), p(imgs), p(sc), p(bx), p(vd),
                                               m, s, i(1 if out_half else 0), i(patch), i(0), p(work), p(out),
                                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("patch", [0, 16])
def test_output_between_guard_words(dtype, patch):
    """the C entry point writes the crops into the middle of a sentinel-filled buffer and nothing around them"""
    name = "sunrgbd"
    nimg, h, w, res = SHAPES[name]
    imgs = _images(name).cuda()
    scene, boxes, valid = crop_cases(name)
    n = len(boxes)
    numel = n * 3 * res * res
    buf = torch.full((numel + 2 * GUARD,), SENTINEL[dtype], dtype=dtype, device="cuda")
    work = torch.empty(nimg * h * w, dtype=torch.int32, device="cuda")
    st = _entry(imgs, scene, boxes, valid, res, n, dtype == torch.float16, patch, work, buf[GUARD:])
    assert st == 0
    torch.cuda.synchronize()
    assert (buf[:GUARD] == SENTINEL[dtype]).all() and (buf[GUARD + numel:] == SENTINEL[dtype]).all()
    exp = _crop(imgs, scene, boxes, valid, res, dtype=dtype, patch=patch)
    assert torch.equal(buf[GUARD:GUARD + numel], exp.reshape(-1))


def test_most_crops_in_one_launch():
    """65535 crops (the grid's limit) at res 16 match fp64 on a sample; one more is refused"""
    nimg, h, w, res, n = MANY
    rng = np.random.default_rng(11)
    imgs = torch.from_numpy(rng.integers(0, 256, (nimg, h, w, 3), dtype=np.uint8)).cuda()
    x0, y0 = rng.integers(0, w - 1, n), rng.integers(0, h - 1, n)
    x1 = np.minimum(x0 + rng.integers(1, w + 1, n), w)
    y1 = np.minimum(y0 + rng.integers(1, h + 1, n), h)
    boxes = np.stack([x0, y0, x1, y1], 1).astype(np.int32)
    scene = rng.integers(0, nimg, n).astype(np.int32)
    valid = rng.random(n) > 0.05
    out = _crop(imgs, scene, boxes, valid, res, dtype=torch.float32)
    sample = np.unique(np.concatenate([np.arange(0, n, 997), [n - 2, n - 1]]))
    _check_against_fp64(out[torch.from_numpy(sample).cuda()], imgs, scene[sample], boxes[sample], valid[sample], res,
                        {})
    with pytest.raises(RuntimeError):
        _crop(imgs, np.zeros(n + 1, np.int32), np.tile(boxes[:1], (n + 1, 1)), np.ones(n + 1, bool), res,
              dtype=torch.float32)


@pytest.mark.parametrize("case", TOO_LARGE)
def test_too_large_is_refused(case):
    nimg, h, w, res = case
    imgs = torch.zeros((nimg, h, w, 3), dtype=torch.uint8, device="cuda")
    box = np.array([[0, 0, w, h]], np.int32)
    with pytest.raises(RuntimeError, match="problem too large for this entry point"):
        _crop(imgs, np.zeros(1, np.int32), box, np.ones(1, bool), res, dtype=torch.float32)


def test_no_crops_launches_nothing():
    """ncrops = 0 returns CODA_OK and touches neither the output nor the workspace (not even the RGBX copy runs)"""
    nimg, h, w, res = SHAPES["small"]
    imgs = _images("small").cuda()
    scene, boxes, valid = crop_cases("small")
    out = torch.full((3 * res * res + 2 * GUARD,), SENTINEL[torch.float32], device="cuda")
    work = torch.full((nimg * h * w,), -123456789, dtype=torch.int32, device="cuda")
    assert _entry(imgs, scene, boxes, valid, res, 0, False, 0, work, out[GUARD:]) == 0
    torch.cuda.synchronize()
    assert (out == SENTINEL[torch.float32]).all() and (work == -123456789).all()
    empty = _crop(imgs, np.zeros(0, np.int32), np.zeros((0, 4), np.int32), np.zeros(0, bool), res, dtype=torch.float32)
    assert empty.shape == (0, 3, res, res)
