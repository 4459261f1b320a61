"""CPU tests (no GPU): the C oracle against hand-checkable cases, against an
independent numpy formulation of the same rules, and against the golden vectors
produced by the reference's own CUDA extension on the GPU
(tests/golden/pointnet2_ref_*.npz, written by tests/golden/make_pointnet2_golden.py)."""
from pathlib import Path

import numpy as np
import pytest

import oracle_pointnet2 as orc
from coda_neurips2023_b200 import synthetic

GOLDEN = Path(__file__).resolve().parent / "golden"


def _bitrev(v: np.ndarray, bits: int) -> np.ndarray:
    out = np.zeros_like(v)
    for i in range(bits):
        out |= ((v >> i) & 1) << (bits - 1 - i)
    return out


def fps_position_space(xyz: np.ndarray, m: int) -> np.ndarray:
    """Independent formulation used by the CUDA kernel: argmax of temp with ties
    broken by the smallest position p = bitrev(k mod bs) * R + k div bs."""
    b, n, _ = xyz.shape
    bs = orc.opt_n_threads(n)
    bits = int(np.log2(bs))
    R = (n + bs - 1) // bs
    k = np.arange(n)
    pos = _bitrev(k % bs, bits) * R + k // bs
    out = np.zeros((b, m), dtype=np.int32)
    for bi in range(b):
        p = xyz[bi].astype(np.float32)
        x, y, z = p[:, 0], p[:, 1], p[:, 2]
        # reference SASS order: FMUL(y,y); FFMA(x,x,.); FFMA(z,z,.)
        mag = np.float32(y * y)
        mag = (x.astype(np.float64) * x.astype(np.float64) + mag.astype(np.float64)).astype(np.float32)  # fma
        mag = (z.astype(np.float64) * z.astype(np.float64) + mag.astype(np.float64)).astype(np.float32)
        valid = ~(mag.astype(np.float64) <= 1e-3)
        temp = np.where(valid, np.float32(1e10), np.float32(-1.0)).astype(np.float32)
        old = 0
        for j in range(1, m):
            d = p - p[old]
            dx, dy, dz = d[:, 0], d[:, 1], d[:, 2]
            # fp32 FMA emulated in float64 (exact for a single product-sum of fp32 operands)
            acc = np.float32(dy * dy)
            acc = (dx.astype(np.float64) * dx + acc.astype(np.float64)).astype(np.float32)
            acc = (dz.astype(np.float64) * dz + acc.astype(np.float64)).astype(np.float32)
            temp = np.where(valid, np.minimum(acc, temp), temp).astype(np.float32)
            if not valid.any():
                old = 0
            else:
                mx = temp[valid].max()
                cand = np.where(valid & (temp == mx))[0]
                old = int(cand[np.argmin(pos[cand])])
            out[bi, j] = old
    return out


def test_opt_n_threads_matches_reference_formula():
    assert orc.opt_n_threads(20000) == 512
    assert orc.opt_n_threads(2048) == 512
    assert orc.opt_n_threads(600) == 512
    assert orc.opt_n_threads(511) == 256
    assert orc.opt_n_threads(5) == 4
    assert orc.opt_n_threads(1) == 1


def test_fps_known_answer_line():
    # points on a line, far from the origin: greedy furthest-point order is forced
    xs = np.array([10.0, 11.0, 12.0, 20.0, 14.0], dtype=np.float32)
    xyz = np.stack([xs, np.full_like(xs, 5.0), np.full_like(xs, 5.0)], -1)[None]
    idx = orc.furthest_point_sampling(xyz, 4)
    # start 0 (x=10) -> furthest x=20 (3) -> then max of min-dist: x=14 (min(4,6)=4) beats 12 (2) -> then 12
    assert idx.tolist() == [[0, 3, 4, 2]]


def test_fps_tie_rule_bit_reversed_thread_wins():
    # SURVEY.md section 7: equal maxima at k=3 and k=130 with bs=512 -> 130 wins
    n = 600
    xyz = np.ones((1, n, 3), dtype=np.float32)
    xyz[0, 3] = xyz[0, 130] = (5.0, 1.0, 1.0)
    idx = orc.furthest_point_sampling(xyz, 2)
    assert idx[0, 1] == 130
    # same stride class (k, k+512): the smaller k wins inside a thread
    xyz = np.ones((1, 1100, 3), dtype=np.float32)
    xyz[0, 7] = xyz[0, 7 + 512] = (5.0, 1.0, 1.0)
    assert orc.furthest_point_sampling(xyz, 2)[0, 1] == 7


def test_fps_skips_points_near_origin_and_all_invalid():
    xyz = np.array([[[2.0, 2.0, 2.0], [0.01, 0.0, 0.0], [3.0, 2.0, 2.0], [0.0, 0.0, 0.0]]], dtype=np.float32)
    idx = orc.furthest_point_sampling(xyz, 3)
    # index 1 and 3 (|p|^2 <= 1e-3) are never selected although they are furthest from point 0
    assert idx.tolist() == [[0, 2, 0]] or idx.tolist() == [[0, 2, 2]]
    assert 1 not in idx and 3 not in idx
    allzero = np.zeros((1, 8, 3), dtype=np.float32)
    assert orc.furthest_point_sampling(allzero, 4).tolist() == [[0, 0, 0, 0]]


@pytest.mark.parametrize("n,m,seed", [(700, 64, 0), (2048, 128, 1), (300, 40, 2), (37, 20, 3)])
def test_fps_literal_simulation_equals_position_space_rule(n, m, seed):
    # heavy duplicates => many exact ties; the literal thread/tree simulation (oracle)
    # and the position-space argmax (what the CUDA kernel computes) must agree
    xyz = synthetic.point_clouds(2, n, seed=seed, dup_frac=0.3, near_origin=min(3, n - 1))
    a = orc.furthest_point_sampling(xyz, m)
    b = fps_position_space(xyz, m)
    assert np.array_equal(a, b)


def test_ball_query_first_hit_padding_and_empty():
    xyz = np.array([[[0, 0, 0], [0.05, 0, 0], [1, 1, 1], [0.1, 0, 0]]], dtype=np.float32)
    new_xyz = np.array([[[0, 0, 0], [5, 5, 5]]], dtype=np.float32)
    idx = orc.ball_query(new_xyz, xyz, 0.2, 4)
    assert idx[0, 0].tolist() == [0, 1, 3, 0]  # three hits in scan order, tail padded with the first
    assert idx[0, 1].tolist() == [0, 0, 0, 0]  # no hit -> zeros
    idx = orc.ball_query(new_xyz, xyz, 0.2, 2)
    assert idx[0, 0].tolist() == [0, 1]        # stops at nsample


def test_ball_query_matches_bruteforce():
    xyz = synthetic.point_clouds(2, 3000, seed=5)
    new_xyz = xyz[:, :200].copy()
    r, ns = 0.3, 16
    idx = orc.ball_query(new_xyz, xyz, r, ns)
    r2 = np.float32(r) * np.float32(r)
    for b in range(2):
        for j in range(0, 200, 17):
            d = new_xyz[b, j][None] - xyz[b]
            d2 = (d.astype(np.float64) ** 2).sum(-1)  # fp64 brute force; skip borderline points
            hits = np.where(d2 < r2 - 1e-6)[0]
            amb = np.where(np.abs(d2 - r2) <= 1e-6)[0]
            if len(amb):
                continue
            exp = list(hits[:ns]) + [hits[0]] * max(0, ns - len(hits)) if len(hits) else [0] * ns
            assert idx[b, j].tolist() == [int(e) for e in exp[:ns]]


def test_three_nn_ties_and_short_known():
    unknown = np.array([[[0, 0, 0]]], dtype=np.float32)
    known = np.array([[[1, 0, 0], [0, 1, 0], [0, 0, 1], [2, 0, 0]]], dtype=np.float32)
    d, i = orc.three_nn(unknown, known)
    assert i[0, 0].tolist() == [0, 1, 2] and d[0, 0].tolist() == [1.0, 1.0, 1.0]  # ascending index on ties
    d, i = orc.three_nn(unknown, known[:, :2])
    assert i[0, 0].tolist() == [0, 1, 0] and np.isinf(d[0, 0, 2])  # unfilled slot: idx 0, dist +inf


def test_group_gather_interpolate_roundtrip():
    rng = np.random.default_rng(0)
    pts = rng.standard_normal((2, 5, 50)).astype(np.float32)
    idx = rng.integers(0, 50, size=(2, 7, 3)).astype(np.int32)
    g = orc.group_points(pts, idx)
    assert g.shape == (2, 5, 7, 3) and g[1, 2, 3, 1] == pts[1, 2, idx[1, 3, 1]]
    go = rng.standard_normal(g.shape).astype(np.float32)
    gg = orc.group_points_grad(go, idx, 50)
    ref = np.zeros((2, 5, 50), dtype=np.float64)
    for b in range(2):
        for j in range(7):
            for s in range(3):
                ref[b, :, idx[b, j, s]] += go[b, :, j, s]
    assert np.allclose(gg, ref, atol=1e-5)
    gi = rng.integers(0, 50, size=(2, 9)).astype(np.int32)
    assert np.array_equal(orc.gather_points(pts, gi)[0, :, 4], pts[0, :, gi[0, 4]])
    w = rng.random((2, 7, 3)).astype(np.float32)
    out = orc.three_interpolate(pts, idx, w)
    exp = sum(np.take_along_axis(pts, np.broadcast_to(idx[:, None, :, t], (2, 5, 7)), 2) * w[:, None, :, t]
              for t in range(3))
    assert np.allclose(out, exp, atol=1e-5)


def test_query_and_group_is_the_unfused_sequence():
    xyz = synthetic.point_clouds(1, 1500, seed=9)
    new_xyz = xyz[:, ::50].copy()
    idx, g = orc.query_and_group_xyz(xyz, new_xyz, 0.4, 8, True)
    assert np.array_equal(idx, orc.ball_query(new_xyz, xyz, 0.4, 8))
    exp = (xyz[0][idx[0]] - new_xyz[0][:, None, :]) * (np.float32(1.0) / np.float32(0.4))
    assert np.array_equal(g[0], np.transpose(exp, (2, 0, 1)).astype(np.float32))


def _golden_files():
    return sorted(GOLDEN.glob("pointnet2_ref_*.npz"))


@pytest.mark.skipif(not _golden_files(), reason="reference-extension golden vectors not generated yet")
@pytest.mark.parametrize("path", _golden_files(), ids=lambda p: p.stem)
def test_oracle_matches_reference_extension_golden(path):
    """Pins the oracle: outputs of the UNMODIFIED reference CUDA extension on the GPU."""
    z = np.load(path)
    xyz = synthetic.point_clouds(int(z["batch"]), int(z["n"]), seed=int(z["seed"]),
                                 dup_frac=float(z["dup_frac"]))
    fps = orc.furthest_point_sampling(xyz, int(z["m"]))
    assert np.array_equal(fps, z["fps_idx"])
    new_xyz = np.take_along_axis(xyz, fps[..., None].astype(np.int64), 1)
    bq = orc.ball_query(new_xyz, xyz, float(z["radius"]), int(z["nsample"]))
    assert np.array_equal(bq, z["ball_idx"])
    known = new_xyz[:, : int(z["nn_known"])]
    d2, nn = orc.three_nn(xyz[:, : int(z["nn_unknown"])], known)
    assert np.array_equal(nn, z["nn_idx"])
    assert np.array_equal(d2, z["nn_dist2"])
