"""The PointNet++ kernels on the H100 at their tile, tie and capacity edges.

Index and copy outputs are compared bit for bit with the C oracle (oracle/pointnet2_oracle.c, which
test_oracle_pointnet2.py pins to the reference extension's own outputs).  Atomically accumulated gradients are compared
with an fp64 scatter, entry by entry, within k * 2^-23 * sum|contribution| for an entry with k contributions, and bit
for bit where every partial sum is exact in fp32.  FPS runs every (instance, cluster width) cell, the generic kernel on
both sides of its boundary and the widening of a forced width; ball query runs on 1, 2 and more tiles, up to the largest
nsample that fits.  test_pointnet2_instances_cpu.py maps these case lists through the launchers' rules
(pointnet2_instances.py) and fails when a cell or an edge is not reached."""
import contextlib
import ctypes
from fractions import Fraction

import numpy as np
import pytest
import torch

import oracle_pointnet2 as orc
import pointnet2_instances as pi
from coda_neurips2023_b200 import synthetic
from coda_neurips2023_b200._lib import lib
from test_oracle_pointnet2 import fps_positions
from test_pointnet2_gpu import cu, ext, ref_ext  # noqa: F401  (ext and ref_ext are fixtures)

pytestmark = pytest.mark.gpu

GUARD = 4                 # guard words on each side of every output (16 bytes: keeps the output 16-byte aligned)
SENTINEL = 0x7FBADBAD     # int32 bits of a NaN: equal to no index and to no grouped coordinate
CODA_ETOOLARGE = -2


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _guarded(count):
    buf = torch.full((count + 2 * GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
    return buf, buf[GUARD:GUARD + count]


def _written(buf, count):
    """The output between the guard words, after checking that every element was written and no guard word was."""
    host = buf.cpu().numpy()
    assert (host[:GUARD] == SENTINEL).all() and (host[GUARD + count:] == SENTINEL).all(), "store outside the output"
    body = host[GUARD:GUARD + count]
    assert (body != SENTINEL).all(), f"{int((body == SENTINEL).sum())} output elements never written"
    return body


def _ok(status):
    assert status == 0, lib().coda_status_string(status).decode()


@contextlib.contextmanager
def _fps_width(width):
    old = lib().coda_fps_set_cluster(width)
    try:
        yield
    finally:
        lib().coda_fps_set_cluster(old)


def _fps(xyz, m, width=0):
    """coda_furthest_point_sampling at a forced cluster width (0: automatic), output between guard words."""
    b, n, _ = xyz.shape
    x = cu(xyz)
    buf, out = _guarded(b * m)
    with _fps_width(width):
        _ok(lib().coda_furthest_point_sampling(b, n, m, _p(x), _p(out), _stream()))
    return _written(buf, b * m).reshape(b, m)


def _near_origin(rng, shape):
    """Points with |p|^2 <= 3 * 0.015^2 < 1e-3, which FPS never selects."""
    return rng.uniform(-0.015, 0.015, size=shape).astype(np.float32)


# ------------------------------------------------------------------ FPS
# (batch, n, m, forced cluster width; 0 = automatic) -> (PPT instance, width) in the comment
FPS_CASES = [
    (3, 37, 20, 1),          # (1, 1): block size 32
    (2, 1024, 200, 1),       # (2, 1)
    (2, 1025, 200, 1),       # (3, 1): one point in the last row
    (2, 2048, 200, 1),       # (4, 1)
    (2, 2559, 200, 1),       # (5, 1)
    (2, 3072, 200, 1),       # (6, 1)
    (2, 3109, 200, 1),       # (8, 1)
    (2, 4097, 200, 1),       # (10, 1)
    (2, 6143, 200, 1),       # (12, 1)
    (2, 6145, 200, 1),       # (16, 1): first n
    (2, 8192, 200, 1),       # (16, 1): last n
    (2, 512, 100, 2),        # (1, 2)
    (2, 1025, 200, 2),       # (2, 2)
    (2, 2560, 200, 2),       # (3, 2)
    (2, 3372, 200, 2),       # (4, 2)
    (2, 4396, 200, 2),       # (5, 2)
    (2, 6144, 200, 2),       # (6, 2)
    (2, 8191, 200, 2),       # (8, 2)
    (2, 10240, 200, 2),      # (10, 2)
    (2, 11813, 200, 2),      # (12, 2)
    (2, 16384, 128, 2),      # (16, 2): last n
    (2, 2048, 200, 4),       # (1, 4)
    (2, 2860, 200, 4),       # (2, 4)
    (2, 5932, 200, 4),       # (3, 4)
    (2, 8192, 200, 4),       # (4, 4)
    (2, 10240, 200, 4),      # (5, 4)
    (2, 11776, 200, 4),      # (6, 4)
    (2, 15872, 128, 4),      # (8, 4)
    (2, 18220, 128, 4),      # (10, 4)
    (2, 20780, 128, 4),      # (12, 4)
    (2, 32768, 128, 4),      # (16, 4): last n
    (3, 37, 20, 8),          # (1, 8): CTAs 1-7 of the cluster hold no point
    (2, 4096, 200, 8),       # (1, 8)
    (2, 8705, 200, 8),       # (3, 8)
    (2, 16383, 128, 8),      # (4, 8)
    (2, 21503, 128, 8),      # (6, 8)
    (2, 24577, 128, 8),      # (8, 8): first n
    (2, 47617, 96, 8),       # (12, 8)
    (2, 49153, 96, 8),       # (16, 8): first n
    (2, 4096, 200, 0),       # automatic: the last n on one CTA -> (8, 1)
    (2, 4097, 200, 0),       # automatic: the first n on a cluster -> (2, 8)
    (2, 20000, 128, 0),      # (5, 8): the pre-encoder's shape
    (2, 40000, 96, 0),       # (10, 8): the ScanNet shape
    (2, 65536, 64, 0),       # (16, 8): the largest register-resident scene
    (2, 65537, 64, 0),       # generic one-CTA kernel
    (2, 8193, 128, 1),       # forced 1 would need 17 points per thread: widened to (3, 8)
    (2, 16385, 128, 2),      # forced 2 would need 17 points per thread: widened to (5, 8)
    (2, 20000, 1, 0),        # m = 1 on a cluster: no round, only the final cluster barrier
    (2, 5000, 2, 2),         # m = 2 on a cluster: one round, no barrier re-armed
    (2, 20000, 3, 0),        # m = 3 on a cluster: the last m with no re-arm
    (2, 5000, 4, 4),         # m = 4: the first re-arm
    (2, 3000, 3100, 2),      # m > n on a cluster: the last rounds tie at distance 0
    (2, 300, 350, 0),        # m > n on one CTA
]


@pytest.mark.parametrize("b,n,m,width", FPS_CASES)
def test_fps_every_instance_and_cluster_width(ext, b, n, m, width):
    xyz = synthetic.point_clouds(b, n, seed=n + 7 * width + m, dup_frac=0.1, near_origin=min(3, n - 1))
    assert np.array_equal(_fps(xyz, m, width), orc.furthest_point_sampling(xyz, m))


@pytest.mark.parametrize("width", [2, 4, 8])
@pytest.mark.parametrize("scene", ["invalid", "equal"])
def test_fps_scenes_without_a_distinct_furthest_point(ext, scene, width):
    """No valid point (every CTA reports none, the exchange falls back to index 0), or every point equal (every round
    is a tie at distance 0 that the smallest position wins)."""
    assert pi.fps_path(5000, width)[1] == width
    rng = np.random.default_rng(width)
    xyz = _near_origin(rng, (2, 5000, 3)) if scene == "invalid" else np.ones((2, 5000, 3), np.float32)
    got = _fps(xyz, 40, width)
    assert np.array_equal(got, orc.furthest_point_sampling(xyz, 40))
    assert not got.any()


@pytest.mark.parametrize("width", [2, 4, 8])
def test_fps_valid_points_in_one_cta_of_the_cluster(ext, width):
    """Only the last CTA of each cluster holds valid points; the others report none every round."""
    n, m = 6000, 150
    assert pi.fps_path(n, width)[1] == width
    owner = pi.fps_cta_of(fps_positions(n), width) == width - 1
    xyz = synthetic.point_clouds(2, n, seed=40 + width, dup_frac=0.05, near_origin=0)
    xyz[:, ~owner] = _near_origin(np.random.default_rng(width), (2, int((~owner).sum()), 3))
    got = _fps(xyz, m, width)
    assert np.array_equal(got, orc.furthest_point_sampling(xyz, m))
    assert owner[got[:, 1:]].all()


def _fma32(a, b, c):
    """fp32 fma(a, b, c) of fp32 operands through fp64; the fp64 value must be exact, so its one rounding is fp32's."""
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    assert Fraction(float(exact)) == exact
    return np.float32(float(exact))


def fps_square_norm(x, y, z):
    """|p|^2 as FPS forms it for the skip test: FMUL y*y, FFMA x, FFMA z, all fp32."""
    x, y, z = np.float32(x), np.float32(y), np.float32(z)
    return _fma32(z, z, _fma32(x, x, y * y))


MAG_BELOW = np.nextafter(np.float32(1e-3), np.float32(0))   # the largest fp32 <= 1e-3
MAG_ABOVE = np.float32(1e-3)                                # > 1e-3 once widened to fp64


def threshold_points(count=6, seed=0):
    """`count` pairs of points one ulp of y apart whose square norm is MAG_BELOW (skipped) and MAG_ABOVE (kept): only
    the comparison of the fp32 square norm, widened to fp64, against the fp64 constant 1e-3 tells them apart."""
    rng = np.random.default_rng(seed)
    below, above = [], []
    up = np.float32(1.0)
    while len(below) < count:
        x, z = rng.uniform(0.008, 0.02, size=2).astype(np.float32) * rng.choice([-1, 1], size=2).astype(np.float32)
        y = np.float32(np.sqrt(1e-3 - float(x) ** 2 - float(z) ** 2))
        while float(fps_square_norm(x, y, z)) > 1e-3:      # compared in fp64, as the kernel does
            y = np.nextafter(y, np.float32(0))
        while float(fps_square_norm(x, np.nextafter(y, up), z)) <= 1e-3:
            y = np.nextafter(y, up)
        y_up = np.nextafter(y, up)
        if fps_square_norm(x, y, z) == MAG_BELOW and fps_square_norm(x, y_up, z) == MAG_ABOVE:
            below.append((x, y, z))
            above.append((x, y_up, z))
    return np.array(below, np.float32), np.array(above, np.float32)


@pytest.mark.parametrize("width", [0, 2, 8])
def test_fps_square_norm_skip_at_its_threshold(ext, width):
    """Points just under the |p|^2 <= 1e-3 skip are never sampled; points just over it are, once m exceeds the
    number of valid points."""
    n, m = 600, 650
    below, above = threshold_points()
    xyz = synthetic.point_clouds(2, n, seed=50, dup_frac=0.0, near_origin=0)
    rng = np.random.default_rng(51)
    skipped = []
    for bi in range(2):
        where = rng.choice(np.arange(1, n), size=2 * len(below), replace=False)
        xyz[bi, where[:len(below)]] = below
        xyz[bi, where[len(below):]] = above
        skipped.append(set(where[:len(below)].tolist()))
    got = _fps(xyz, m, width)
    assert np.array_equal(got, orc.furthest_point_sampling(xyz, m))
    for bi in range(2):
        assert set(got[bi].tolist()) == set(range(n)) - skipped[bi]


# ------------------------------------------------------------------ ball query / fused grouping
def _ball_query(xyz, new_xyz, radius, ns, group=False, normalize=False):
    """coda_ball_query or coda_query_and_group_xyz, every output between guard words."""
    b, n, _ = xyz.shape
    m = new_xyz.shape[1]
    x, c = cu(xyz), cu(new_xyz)
    ib, idx = _guarded(b * m * ns)
    i, f = ctypes.c_int, ctypes.c_float
    if not group:
        _ok(lib().coda_ball_query(i(b), i(n), i(m), f(radius), i(ns), _p(c), _p(x), _p(idx), _stream()))
        return _written(ib, b * m * ns).reshape(b, m, ns)
    gb, g = _guarded(b * 3 * m * ns)
    _ok(lib().coda_query_and_group_xyz(i(b), i(n), i(m), f(radius), i(ns), i(int(normalize)), _p(x), _p(c), _p(idx),
                                       _p(g), _stream()))
    grouped = _written(gb, b * 3 * m * ns).view(np.float32).reshape(b, 3, m, ns)
    return _written(ib, b * m * ns).reshape(b, m, ns), grouped


def _bq_scene(b, n, m, radius, seed, offset=0.0):
    """Room scene whose ball centres sit on clusters of consecutive indices around every tile boundary (and at random
    indices), with every fifth centre far from all points (no hit)."""
    rng = np.random.default_rng(seed)
    xyz = synthetic.point_clouds(b, n, seed=seed, dup_frac=0.05, near_origin=0).astype(np.float64)
    new = np.empty((b, m, 3))
    bounds = [t * pi.BQ_TILE + d for t in range(1, pi.bq_tiles(n)) for d in (-1, 0)]
    for bi in range(b):
        for j in range(m):
            if j % 5 == 4:
                new[bi, j] = (40.0, 40.0, 40.0 + j)
                continue
            a = bounds[j % len(bounds)] if bounds and j % 5 < 2 else int(rng.integers(0, n))
            new[bi, j] = xyz[bi, a] + rng.uniform(-0.1, 0.1, 3) * radius
            lo, hi = max(0, a - 3), min(n, a + 3)
            xyz[bi, lo:hi] = new[bi, j] + rng.uniform(-0.5, 0.5, (hi - lo, 3)) * radius
    return (xyz + offset).astype(np.float32), (new + offset).astype(np.float32)


# (batch, n, m, radius, nsample, offset of the whole scene from the origin)
BQ_CASES = [
    (2, 2047, 37, 0.3, 33, 0.0),       # one short tile; 5 of the last CTA's 8 warps active
    (2, 2048, 64, 0.3, 31, 0.0),       # one full tile
    (2, 2049, 29, 0.5, 64, 0.0),       # two tiles, the second holding one point
    (2, 4097, 100, 0.4, 32, 0.0),      # three tiles at the masked encoder's radius and nsample
    (1, 4097, 13, 0.3, 1, 0.0),        # nsample 1: warps finish on their first hit, CTAs before the last tile
    (2, 20000, 203, 0.2, 64, 0.0),     # ten tiles at the pre-encoder's radius and nsample
    (2, 4097, 45, 0.4, 33, 1000.0),    # 1 km from the origin
    (2, 5000, 21, 0.05, 200, 0.0),     # small balls: short hit lists padded over seven passes of each lane
    (1, 6000, 13, 2.0, 5632, 0.0),     # the largest nsample whose hit lists fit in shared memory
]


@pytest.mark.parametrize("b,n,m,radius,ns,offset", BQ_CASES)
def test_ball_query_and_fused_grouping_vs_oracle(ext, b, n, m, radius, ns, offset):
    xyz, new = _bq_scene(b, n, m, radius, seed=n + m + ns, offset=offset)
    exp = orc.ball_query(new, xyz, radius, ns)
    assert not exp[:, 4::5].any()                                       # the far centres: no hit, zeros
    assert (exp[..., -1] == exp[..., 0]).any()                          # rows padded with their first hit
    if pi.bq_tiles(n) > 1 and ns > 1:                                   # hit lists spanning a tile boundary
        assert (exp[..., 0] // pi.BQ_TILE != exp.max(-1) // pi.BQ_TILE).any()
    assert np.array_equal(_ball_query(xyz, new, radius, ns), exp)
    for normalize in (False, True):
        idx, g = _ball_query(xyz, new, radius, ns, group=True, normalize=normalize)
        eidx, eg = orc.query_and_group_xyz(xyz, new, radius, ns, normalize)
        assert np.array_equal(idx, eidx)
        assert np.array_equal(g.view(np.int32), eg.view(np.int32))


def _sphere_scene():
    """A centre, points exactly on its sphere of radius 5/8 (every coordinate and every step of the fp32 distance is
    exact, so d2 == r^2), points 2^-20 inside and outside it, and far filler, over two tiles."""
    r = 0.625
    c = np.array([1.0, 2.0, 0.5])
    on = np.array([(s * a, t * b_, 0.0) for a, b_ in ((0.375, 0.5), (0.5, 0.375)) for s in (1, -1) for t in (1, -1)]
                  + [(0.0, 0.375, 0.5), (0.0, -0.5, -0.375), (0.625, 0.0, 0.0), (0.0, 0.0, -0.625)])
    inside = on * (1 - 2.0 ** -20 / r)
    outside = on * (1 + 2.0 ** -20 / r)
    n = 2100
    xyz = synthetic.point_clouds(1, n, seed=60, near_origin=0).astype(np.float64) + (20.0, 0.0, 0.0)
    at_on = np.r_[0:6, 2044:2050]                     # first scanned, and across the tile boundary
    at_in = np.r_[6:10, 2036:2044]
    at_out = np.r_[10:22]
    xyz[0, at_on], xyz[0, at_in], xyz[0, at_out] = c + on, c + inside, c + outside
    new = np.tile(c, (1, 11, 1))                      # 11 identical centres: three warps of the second CTA idle
    return xyz.astype(np.float32), new.astype(np.float32), r, at_on, at_in


def test_ball_query_hit_rule_is_strict_at_r_squared(ext):
    xyz, new, r, at_on, at_in = _sphere_scene()
    d = xyz[0, at_on] - new[0, 0]
    assert all(fps_square_norm(*v) == np.float32(r) * np.float32(r) for v in d)   # d2 == r^2 in the kernel's order
    exp = orc.ball_query(new, xyz, r, 64)
    assert set(exp[0, 0].tolist()) == set(at_in.tolist())
    assert np.array_equal(_ball_query(xyz, new, r, 64), exp)
    for normalize in (False, True):
        idx, g = _ball_query(xyz, new, r, 64, group=True, normalize=normalize)
        eidx, eg = orc.query_and_group_xyz(xyz, new, r, 64, normalize)
        assert np.array_equal(idx, eidx) and np.array_equal(g.view(np.int32), eg.view(np.int32))


def test_ball_query_on_an_empty_scene(ext):
    empty = np.zeros((2, 0, 3), np.float32)
    new = synthetic.point_clouds(2, 13, seed=70)
    assert not _ball_query(empty, new, 0.3, 33).any()
    with pytest.raises(RuntimeError, match="invalid argument"):
        ext.query_and_group_xyz(cu(empty), cu(new), 0.3, 33, True)


def test_nsample_beyond_shared_memory_is_refused(ext):
    ns = pi.bq_max_nsample() + 1
    xyz, new = cu(synthetic.point_clouds(1, 100, seed=71)), cu(synthetic.point_clouds(1, 9, seed=72))
    i, f = ctypes.c_int, ctypes.c_float
    idx = torch.empty(9 * ns, dtype=torch.int32, device="cuda")
    g = torch.empty(3 * 9 * ns, dtype=torch.float32, device="cuda")
    assert lib().coda_ball_query(i(1), i(100), i(9), f(0.3), i(ns), _p(new), _p(xyz), _p(idx), _stream()) \
        == CODA_ETOOLARGE
    assert lib().coda_query_and_group_xyz(i(1), i(100), i(9), f(0.3), i(ns), i(1), _p(xyz), _p(new), _p(idx), _p(g),
                                          _stream()) == CODA_ETOOLARGE
    with pytest.raises(RuntimeError, match="too large"):
        ext.ball_query(new, xyz, 0.3, ns)
    with pytest.raises(RuntimeError, match="too large"):
        ext.query_and_group_xyz(xyz, new, 0.3, ns, True)


# (batch, n, m, radius, nsample): the masked encoder's interim down-sampling and the ScanNet pre-encoder
STEP_BALLS = [(8, 2048, 1024, 0.4, 32), (2, 40000, 2048, 0.2, 64)]


@pytest.mark.parametrize("b,n,m,radius,ns", STEP_BALLS)
def test_fused_query_and_group_equals_torch_ops_at_step_shapes(ext, b, n, m, radius, ns):
    """pointnet2_utils.py:331-349 executed with torch CUDA ops, bit for bit."""
    xyz = cu(synthetic.point_clouds(b, n, seed=m))
    inds = ext.furthest_point_sampling(xyz, m)
    new_xyz = ext.gather_points(xyz.transpose(1, 2).contiguous(), inds).transpose(1, 2).contiguous()
    for normalize in (True, False):
        idx = ext.ball_query(new_xyz, xyz, radius, ns)
        g = ext.group_points(xyz.transpose(1, 2).contiguous(), idx)
        g -= new_xyz.transpose(1, 2).unsqueeze(-1)
        if normalize:
            g /= radius
        idx2, g2 = ext.query_and_group_xyz(xyz, new_xyz, radius, ns, normalize)
        assert torch.equal(idx, idx2) and torch.equal(g.view(torch.int32), g2.view(torch.int32))


# ------------------------------------------------------------------ gather / group and their gradients
def _scatter_check(got, values, targets, size, exact=False):
    """got (fp32) against the fp64 sum of `values` per target: within k * 2^-23 * sum|value| for a target with k
    values, or bit for bit when every partial sum is exact in fp32."""
    v = values.astype(np.float64).ravel()
    t = targets.ravel()
    s = np.bincount(t, weights=v, minlength=size)
    a = np.bincount(t, weights=np.abs(v), minlength=size)
    k = np.bincount(t, minlength=size)
    got = got.astype(np.float64).ravel()
    if exact:
        assert np.array_equal(got, s)
        return
    err = np.abs(got - s)
    bound = k * 2.0 ** -23 * a
    worst = int(np.argmax(err - bound))
    assert (err <= bound).all(), f"entry {worst}: |{got[worst]} - {s[worst]}| > {bound[worst]} ({k[worst]} terms)"


def _grad_values(rng, shape, exact):
    """Standard normal, or multiples of 2^-8 no larger than 1/4, whose fp32 partial sums are all exact."""
    if exact:
        return (rng.integers(-64, 65, size=shape) * 2.0 ** -8).astype(np.float32)
    return rng.standard_normal(shape).astype(np.float32)


def _group_indices(b, n, npoints, ns, source, seed):
    """Indices from a real ball query (rows padded with their first hit), or every index the same point."""
    if source == "one":
        return np.broadcast_to((np.arange(b) * 577 % n)[:, None, None], (b, npoints, ns)).astype(np.int32).copy()
    xyz = synthetic.point_clouds(b, n, seed=seed)
    new = np.take_along_axis(xyz, orc.furthest_point_sampling(xyz, npoints)[..., None].astype(np.int64), 1)
    idx = orc.ball_query(new, xyz, 0.4, ns)
    assert (idx[..., -1] == idx[..., 0]).any()
    return idx


# (batch, channels, n, npoints, nsample, index source)
GROUP_CASES = [
    (2, 1, 777, 37, 5, "ball"),
    (8, 3, 2048, 1000, 33, "ball"),      # 33000 elements per channel: two slices of 2 and 1 channels
    (8, 5, 2048, 1000, 33, "ball"),      # slices of 3 and 2
    (2, 259, 4097, 100, 7, "ball"),      # 130 slices, the last of one channel
    (4, 5, 3000, 333, 17, "one"),        # 5661 contributions to one point per channel
    (8, 256, 2048, 1024, 32, "ball"),    # the masked encoder's interim down-sampling
]


@pytest.mark.parametrize("b,c,n,npoints,ns,source", GROUP_CASES)
def test_group_points_and_gradient(ext, b, c, n, npoints, ns, source):
    rng = np.random.default_rng(n + c)
    idx = _group_indices(b, n, npoints, ns, source, seed=n + c)
    pts = rng.standard_normal((b, c, n)).astype(np.float32)
    di = cu(idx)
    got = ext.group_points(cu(pts), di).cpu().numpy()
    assert np.array_equal(got.view(np.int32), orc.group_points(pts, idx).view(np.int32))
    for exact in (False, True):
        go = _grad_values(rng, (b, c, npoints, ns), exact)
        g = ext.group_points_grad(cu(go), di, n).cpu().numpy()
        for bi in range(b):
            _scatter_check(g[bi], go[bi], np.arange(c)[:, None] * n + idx[bi].reshape(1, -1), c * n, exact)


# (batch, channels, n, m, index source)
GATHER_CASES = [(2, 1, 2049, 257, "fps"), (2, 259, 4097, 1000, "fps"), (3, 5, 3000, 300, "one")]


@pytest.mark.parametrize("b,c,n,m,source", GATHER_CASES)
def test_gather_points_and_gradient(ext, b, c, n, m, source):
    rng = np.random.default_rng(n + c)
    if source == "one":
        idx = np.broadcast_to((np.arange(b) * 577 % n)[:, None], (b, m)).astype(np.int32).copy()
    else:
        idx = orc.furthest_point_sampling(synthetic.point_clouds(b, n, seed=n), m)
    pts = rng.standard_normal((b, c, n)).astype(np.float32)
    got = ext.gather_points(cu(pts), cu(idx)).cpu().numpy()
    assert np.array_equal(got.view(np.int32), orc.gather_points(pts, idx).view(np.int32))
    targets = np.arange(c)[:, None] * n + idx[:, None, :]
    for exact in (False, True):
        go = _grad_values(rng, (b, c, m), exact)
        g = ext.gather_points_grad(cu(go), cu(idx), n).cpu().numpy()
        for bi in range(b):
            _scatter_check(g[bi], go[bi], targets[bi], c * n, exact)


# ------------------------------------------------------------------ three_nn / three_interpolate
def _nn_scene(b, n, m, seed):
    """Known points with exact duplicates, one of them at 1023 and 1024 (and 2048) across the 1024-point tile; the
    first unknowns sit on or next to known points so that ties decide the order."""
    known = synthetic.point_clouds(b, m, seed=seed, dup_frac=0.1, near_origin=0)
    unknown = synthetic.point_clouds(b, n, seed=seed + 1, near_origin=0)
    if m > 1024:
        known[:, 1024] = known[:, 1023]
    if m > 2048:
        known[:, 2048] = known[:, 1023]
    if m:
        rng = np.random.default_rng(seed)
        src = np.r_[np.full(20, min(m - 1, 1023)), rng.integers(0, m, 40)]
        jitter = rng.uniform(-1e-3, 1e-3, (60, 3)).astype(np.float32)
        jitter[::3] = 0
        unknown[:, :60] = known[:, src] + jitter
    return unknown, known


# (batch, unknowns, known points)
NN_CASES = [(2, 300, 0), (2, 300, 1), (2, 300, 2), (2, 300, 3), (2, 1000, 1023), (2, 1000, 1024), (2, 1000, 1025),
            (2, 777, 2049)]


@pytest.mark.parametrize("b,n,m", NN_CASES)
def test_three_nn_tiles_ties_and_short_known_sets(ext, b, n, m):
    unknown, known = _nn_scene(b, n, m, seed=n + m)
    d2, idx = ext.three_nn(cu(unknown), cu(known))
    ed2, eidx = orc.three_nn(unknown, known)
    if m > 1024:   # the duplicate pair across the tile boundary: the lower index first
        assert ((eidx[..., 0] == 1023) & (eidx[..., 1] == 1024)).any()
    assert np.array_equal(idx.cpu().numpy(), eidx)
    assert np.array_equal(d2.cpu().numpy().view(np.int32), ed2.view(np.int32))


# (batch, channels, unknowns, known points)
INTERP_CASES = [(2, 1, 300, 1), (2, 5, 300, 3), (2, 259, 1000, 2049), (2, 3, 100000, 1025), (2, 5, 100000, 1025)]


@pytest.mark.parametrize("b,c,n,m", INTERP_CASES)
def test_three_interpolate_and_gradient(ext, b, c, n, m):
    unknown, known = _nn_scene(b, n, m, seed=n + m)
    _, idx = orc.three_nn(unknown, known)
    rng = np.random.default_rng(c + m)
    feats = rng.standard_normal((b, c, m)).astype(np.float32)
    w = rng.random((b, n, 3)).astype(np.float32)
    di = cu(idx)
    got = ext.three_interpolate(cu(feats), di, cu(w)).cpu().numpy()
    assert np.array_equal(got.view(np.int32), orc.three_interpolate(feats, idx, w).view(np.int32))
    targets = np.arange(c)[:, None] * m + idx.reshape(b, 1, -1)             # (b, c, n * 3)
    for exact in (False, True):
        go = _grad_values(rng, (b, c, n), exact)
        if exact:   # weights of 4 bits: every product and partial sum is exact in fp32
            w = (rng.integers(0, 17, size=(b, n, 3)) / 16.0).astype(np.float32)
        g = ext.three_interpolate_grad(cu(go), di, cu(w), m).cpu().numpy()
        contrib = go[:, :, :, None].astype(np.float64) * w[:, None].astype(np.float64)     # (b, c, n, 3)
        for bi in range(b):
            _scatter_check(g[bi], contrib[bi], targets[bi], c * m, exact)


# ------------------------------------------------------------------ reference extension
def test_fps_cells_and_ball_query_edges_vs_reference_extension(ext, ref_ext):
    """The new FPS cells and ball-query edges against the UNMODIFIED reference extension on the same GPU."""
    for b, n, m, width in FPS_CASES:
        xyz = synthetic.point_clouds(b, n, seed=n + 7 * width + m, dup_frac=0.1, near_origin=min(3, n - 1))
        assert np.array_equal(_fps(xyz, m, width), ref_ext.furthest_point_sampling(cu(xyz), m).cpu().numpy()), \
            f"FPS differs from the reference at n={n}, m={m}, width={width}"
    scenes = [(*_bq_scene(b, n, m, r, seed=n + m + ns, offset=off), r, ns) for b, n, m, r, ns, off in BQ_CASES]
    scenes.append(_sphere_scene()[:3] + (64,))
    for xyz, new, r, ns in scenes:
        assert np.array_equal(_ball_query(xyz, new, r, ns),
                              ref_ext.ball_query(cu(new), cu(xyz), r, ns).cpu().numpy()), \
            f"ball query differs from the reference at n={xyz.shape[1]}, nsample={ns}"
