"""GPU parity tests: the sm_90a kernels (through the C-ABI / `_ext` binding)
against the CPU oracle, against the reference's own CUDA extension when its
build travelled with the snapshot (oracle/_ref), and against the golden vectors.
Bar: bit-exact for indices and for pure copies; 1e-5 for atomically accumulated
gradients (the reference's own accumulation order is unspecified)."""
import importlib
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_pointnet2 as orc
from coda_neurips2023_b200 import synthetic

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"


@pytest.fixture(scope="module")
def ext(built_lib):
    from coda_neurips2023_b200.pointnet2 import _ext

    return _ext


@pytest.fixture(scope="module")
def ref_ext():
    """The reference's unmodified extension, compiled by oracle/build_ref_ext.py."""
    so = ROOT / "oracle" / "_ref" / "pointnet2" / "_ext.so"
    if not so.exists():
        pytest.skip("oracle/_ref/pointnet2/_ext.so not built")
    sys.path.insert(0, str(ROOT / "oracle" / "_ref"))
    try:
        return importlib.import_module("pointnet2._ext")
    finally:
        sys.path.pop(0)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------ FPS
FPS_CASES = [
    # (batch, n, m, seed, dup_frac)
    (8, 20000, 2048, 0, 0.01),   # SUN RGB-D pre-encoder call (cluster of 8, 5 points / thread)
    (8, 2048, 256, 1, 0.01),     # query sampling call (single CTA)
    (2, 40000, 2048, 2, 0.02),   # ScanNet shape
    (3, 37, 20, 3, 0.3), (3, 300, 40, 4, 0.3), (2, 511, 64, 5, 0.2), (2, 512, 64, 6, 0.2),
    (2, 513, 64, 7, 0.2), (2, 1000, 100, 8, 0.5), (2, 4097, 128, 9, 0.1), (1, 1, 1, 10, 0.0),
    (2, 5, 5, 11, 0.0),
]


@pytest.mark.parametrize("b,n,m,seed,dup", FPS_CASES)
def test_fps_bit_exact_vs_oracle(ext, b, n, m, seed, dup):
    xyz = synthetic.point_clouds(b, n, seed=seed, dup_frac=dup, near_origin=min(3, n - 1))
    got = ext.furthest_point_sampling(cu(xyz), m).cpu().numpy()
    assert got.dtype == np.int32 and got.shape == (b, m)
    assert np.array_equal(got, orc.furthest_point_sampling(xyz, m))


@pytest.mark.parametrize("cl", [1, 2, 4, 8])
def test_fps_every_cluster_width(ext, cl):
    from coda_neurips2023_b200._lib import lib

    xyz = synthetic.point_clouds(3, 5000, seed=20 + cl, dup_frac=0.2)
    exp = orc.furthest_point_sampling(xyz, 300)
    old = lib().coda_fps_set_cluster(cl)
    try:
        got = ext.furthest_point_sampling(cu(xyz), 300).cpu().numpy()
    finally:
        lib().coda_fps_set_cluster(old)
    assert np.array_equal(got, exp)


def test_fps_generic_fallback_for_huge_scenes(ext):
    xyz = synthetic.point_clouds(2, 70000, seed=31, dup_frac=0.05)
    got = ext.furthest_point_sampling(cu(xyz), 48).cpu().numpy()
    assert np.array_equal(got, orc.furthest_point_sampling(xyz, 48))


def test_fps_degenerate_scenes(ext):
    allzero = np.zeros((2, 100, 3), dtype=np.float32)  # every point is skipped -> index 0 forever
    assert np.array_equal(ext.furthest_point_sampling(cu(allzero), 10).cpu().numpy(), np.zeros((2, 10), np.int32))
    same = np.ones((1, 700, 3), dtype=np.float32)      # all ties at distance 0
    assert np.array_equal(ext.furthest_point_sampling(cu(same), 16).cpu().numpy(),
                          orc.furthest_point_sampling(same, 16))
    assert ext.furthest_point_sampling(cu(same), 0).shape == (1, 0)


def test_fps_full_size_properties(ext):
    """Size-independent checks at BASELINE size (8 x 20 000 -> 2048): indices are distinct, the first is 0, and
    the greedy invariant holds -- sample j is THE point farthest from samples 0..j-1 (checked at every 97th
    round in fp64), so the max-min distance never increases along the sequence."""
    xyz = synthetic.point_clouds(8, 20000, seed=77, dup_frac=0.0, near_origin=0)
    idx = ext.furthest_point_sampling(cu(xyz), 2048).cpu().numpy().astype(np.int64)
    assert (idx[:, 0] == 0).all() and idx.min() >= 0 and idx.max() < 20000
    for b in range(8):
        assert len(np.unique(idx[b])) == 2048
        pts = xyz[b].astype(np.float64)
        mind = np.full(20000, np.inf)
        prev = np.inf
        for j in range(1, 2048):
            mind = np.minimum(mind, ((pts - pts[idx[b, j - 1]]) ** 2).sum(-1))
            if j % 97 == 1:
                chosen = mind[idx[b, j]]
                assert chosen >= mind.max() * (1 - 1e-5), (b, j)      # farthest point (fp32 vs fp64 slack)
                assert chosen <= prev * (1 + 1e-5), (b, j)            # max-min distance is non-increasing
                prev = chosen


# ------------------------------------------------------------------ ball query / grouping
@pytest.mark.parametrize("b,n,m,r,ns,seed", [
    (8, 20000, 2048, 0.2, 64, 0), (2, 3000, 256, 0.3, 16, 1), (2, 500, 100, 0.05, 8, 2),
    (1, 2050, 7, 5.0, 32, 3), (2, 40000, 1024, 0.4, 32, 4), (1, 33, 33, 0.5, 3, 5),
])
def test_ball_query_bit_exact_vs_oracle(ext, b, n, m, r, ns, seed):
    xyz = synthetic.point_clouds(b, n, seed=seed)
    fps = orc.furthest_point_sampling(xyz, m) if n <= 5000 else \
        ext.furthest_point_sampling(cu(xyz), m).cpu().numpy()
    new_xyz = np.take_along_axis(xyz, fps[..., None].astype(np.int64), 1)
    got = ext.ball_query(cu(new_xyz), cu(xyz), r, ns).cpu().numpy()
    exp = orc.ball_query(new_xyz, xyz, r, ns)
    assert np.array_equal(got, exp)
    idx2, grouped = ext.query_and_group_xyz(cu(xyz), cu(new_xyz), r, ns, True)
    eidx, egrouped = orc.query_and_group_xyz(xyz, new_xyz, r, ns, True)
    assert np.array_equal(idx2.cpu().numpy(), eidx)
    assert np.array_equal(grouped.cpu().numpy(), egrouped)


def test_fused_query_and_group_equals_torch_op_sequence(ext):
    """pointnet2_utils.py:331-349 executed with torch CUDA ops, bit for bit."""
    xyz = cu(synthetic.point_clouds(4, 20000, seed=3))
    inds = ext.furthest_point_sampling(xyz, 512)
    new_xyz = ext.gather_points(xyz.transpose(1, 2).contiguous(), inds).transpose(1, 2).contiguous()
    for normalize in (True, False):
        idx = ext.ball_query(new_xyz, xyz, 0.2, 64)
        g = ext.group_points(xyz.transpose(1, 2).contiguous(), idx)
        g -= new_xyz.transpose(1, 2).unsqueeze(-1)
        if normalize:
            g /= 0.2
        idx2, g2 = ext.query_and_group_xyz(xyz, new_xyz, 0.2, 64, normalize)
        assert torch.equal(idx, idx2) and torch.equal(g, g2)


def test_ball_query_full_size_properties(ext):
    xyz = synthetic.point_clouds(8, 20000, seed=5)
    x = cu(xyz)
    inds = ext.furthest_point_sampling(x, 2048)
    new_xyz = torch.gather(x, 1, inds.long()[..., None].expand(-1, -1, 3)).contiguous()
    idx = ext.ball_query(new_xyz, x, 0.2, 64).long()
    assert idx.min() >= 0 and idx.max() < 20000
    pts = torch.gather(x[:, None].expand(-1, 2048, -1, -1), 2, idx[..., None].expand(-1, -1, -1, 3))
    d2 = ((pts - new_xyz[:, :, None]) ** 2).sum(-1)
    assert (d2 < 0.2 * 0.2 + 1e-6).all()           # every returned point is inside the ball
    # each centre is itself a scene point => never empty; hits ascend until the padding starts
    first = idx[..., :1]
    body = idx[..., 1:] - idx[..., :-1]
    assert ((body > 0) | (idx[..., 1:] == first)).all()


# ------------------------------------------------------------------ gather / group / interpolate
def test_gather_group_and_grads_vs_oracle(ext):
    rng = np.random.default_rng(0)
    pts = rng.standard_normal((3, 19, 777)).astype(np.float32)
    gi = rng.integers(0, 777, size=(3, 300)).astype(np.int32)
    assert np.array_equal(ext.gather_points(cu(pts), cu(gi)).cpu().numpy(), orc.gather_points(pts, gi))
    go = rng.standard_normal((3, 19, 300)).astype(np.float32)
    np.testing.assert_allclose(ext.gather_points_grad(cu(go), cu(gi), 777).cpu().numpy(),
                               orc.gather_points_grad(go, gi, 777), atol=1e-5)
    idx = rng.integers(0, 777, size=(3, 50, 9)).astype(np.int32)
    assert np.array_equal(ext.group_points(cu(pts), cu(idx)).cpu().numpy(), orc.group_points(pts, idx))
    go = rng.standard_normal((3, 19, 50, 9)).astype(np.float32)
    np.testing.assert_allclose(ext.group_points_grad(cu(go), cu(idx), 777).cpu().numpy(),
                               orc.group_points_grad(go, idx, 777), atol=1e-5)


def test_three_nn_and_interpolate_vs_oracle(ext):
    xyz = synthetic.point_clouds(2, 5000, seed=11, dup_frac=0.2)
    unknown, known = xyz[:, :3000], xyz[:, 3000:4500]
    d2, idx = ext.three_nn(cu(unknown), cu(known))
    ed2, eidx = orc.three_nn(unknown, known)
    assert np.array_equal(idx.cpu().numpy(), eidx) and np.array_equal(d2.cpu().numpy(), ed2)
    d2s, idxs = ext.three_nn(cu(unknown[:, :10]), cu(known[:, :2]))  # m < 3
    ed2s, eidxs = orc.three_nn(unknown[:, :10], known[:, :2])
    assert np.array_equal(idxs.cpu().numpy(), eidxs) and np.array_equal(d2s.cpu().numpy(), ed2s)
    rng = np.random.default_rng(1)
    feats = rng.standard_normal((2, 33, 1500)).astype(np.float32)
    w = rng.random((2, 3000, 3)).astype(np.float32)
    out = ext.three_interpolate(cu(feats), idx, cu(w)).cpu().numpy()
    assert np.array_equal(out, orc.three_interpolate(feats, eidx, w))
    go = rng.standard_normal((2, 33, 3000)).astype(np.float32)
    np.testing.assert_allclose(ext.three_interpolate_grad(cu(go), idx, cu(w), 1500).cpu().numpy(),
                               orc.three_interpolate_grad(go, eidx, w, 1500), atol=2e-5)


# ------------------------------------------------------------------ reference extension
def test_every_op_vs_reference_extension(ext, ref_ext):
    """Our kernels against the UNMODIFIED reference extension on the same GPU."""
    for (b, n, m, seed) in [(8, 20000, 2048, 0), (4, 2048, 256, 1), (2, 700, 128, 2)]:
        xyz = cu(synthetic.point_clouds(b, n, seed=seed, dup_frac=0.05))
        ours, ref = ext.furthest_point_sampling(xyz, m), ref_ext.furthest_point_sampling(xyz, m)
        assert torch.equal(ours, ref), f"FPS differs from the reference at n={n}"
        flipped = xyz.transpose(1, 2).contiguous()
        new_o, new_r = ext.gather_points(flipped, ours), ref_ext.gather_points(flipped, ref)
        assert torch.equal(new_o, new_r)
        new_xyz = new_o.transpose(1, 2).contiguous()
        io, ir = ext.ball_query(new_xyz, xyz, 0.2, 64), ref_ext.ball_query(new_xyz, xyz, 0.2, 64)
        assert torch.equal(io, ir)
        assert torch.equal(ext.group_points(flipped, io), ref_ext.group_points(flipped, ir))
        go = torch.randn(b, 3, m, 64, device="cuda")
        torch.testing.assert_close(ext.group_points_grad(go, io, n), ref_ext.group_points_grad(go, ir, n),
                                   atol=1e-4, rtol=1e-5)
        g1 = torch.randn(b, 3, m, device="cuda")
        torch.testing.assert_close(ext.gather_points_grad(g1, ours, n), ref_ext.gather_points_grad(g1, ref, n),
                                   atol=1e-5, rtol=1e-5)
        (do, no), (dr, nr) = ext.three_nn(xyz[:, :1500].contiguous(), new_xyz), \
            ref_ext.three_nn(xyz[:, :1500].contiguous(), new_xyz)
        assert torch.equal(no, nr) and torch.equal(do, dr)
        feats = torch.randn(b, 16, m, device="cuda")
        w = torch.rand(b, min(n, 1500), 3, device="cuda")
        assert torch.equal(ext.three_interpolate(feats, no, w), ref_ext.three_interpolate(feats, nr, w))
        g2 = torch.randn(b, 16, min(n, 1500), device="cuda")
        torch.testing.assert_close(ext.three_interpolate_grad(g2, no, w, m),
                                   ref_ext.three_interpolate_grad(g2, nr, w, m), atol=1e-4, rtol=1e-5)


def _golden_files():
    return sorted(GOLDEN.glob("pointnet2_ref_*.npz"))


@pytest.mark.skipif(not _golden_files(), reason="golden vectors not generated yet")
@pytest.mark.parametrize("path", _golden_files(), ids=lambda p: p.stem)
def test_kernels_match_committed_golden(ext, path):
    z = np.load(path)
    xyz = synthetic.point_clouds(int(z["batch"]), int(z["n"]), seed=int(z["seed"]), dup_frac=float(z["dup_frac"]))
    x = cu(xyz)
    fps = ext.furthest_point_sampling(x, int(z["m"]))
    assert np.array_equal(fps.cpu().numpy(), z["fps_idx"])
    new_xyz = torch.gather(x, 1, fps.long()[..., None].expand(-1, -1, 3)).contiguous()
    assert np.array_equal(ext.ball_query(new_xyz, x, float(z["radius"]), int(z["nsample"])).cpu().numpy(),
                          z["ball_idx"])
    d2, nn = ext.three_nn(x[:, : int(z["nn_unknown"])].contiguous(), new_xyz[:, : int(z["nn_known"])].contiguous())
    assert np.array_equal(nn.cpu().numpy(), z["nn_idx"]) and np.array_equal(d2.cpu().numpy(), z["nn_dist2"])


# ------------------------------------------------------------------ error behaviour / autograd
def test_error_behaviour_matches_reference_contract(ext):
    with pytest.raises(RuntimeError, match="CPU not supported"):
        ext.furthest_point_sampling(torch.zeros(1, 10, 3), 2)
    x = torch.zeros(1, 3, 10, device="cuda").transpose(1, 2)  # non-contiguous
    with pytest.raises(RuntimeError, match="contiguous"):
        ext.furthest_point_sampling(x, 2)
    with pytest.raises(RuntimeError, match="float"):
        ext.furthest_point_sampling(torch.zeros(1, 10, 3, device="cuda", dtype=torch.float64), 2)
    with pytest.raises(RuntimeError, match="int"):
        ext.gather_points(torch.zeros(1, 3, 10, device="cuda"), torch.zeros(1, 4, device="cuda", dtype=torch.int64))


def test_autograd_functions_and_sa_module(ext):
    from coda_neurips2023_b200.pointnet2 import pointnet2_utils as pu
    from coda_neurips2023_b200.pointnet2.pointnet2_modules import PointnetSAModuleVotes

    torch.manual_seed(0)
    # the reference's only unit test: gradcheck of three_interpolate (pointnet2_test.py:15-27)
    feats = torch.randn(1, 2, 4, device="cuda", requires_grad=True)
    idx = torch.tensor([[[0, 1, 2], [1, 2, 3]]], device="cuda", dtype=torch.int32)
    w = torch.tensor([[[1.0, 1.0, 1.0], [2.0, 2.0, 2.0]]], device="cuda")
    out = pu.three_interpolate(feats, idx, w)
    out.sum().backward()
    exp = torch.zeros(1, 2, 4, device="cuda")
    exp[..., 0] = 1; exp[..., 1] = 3; exp[..., 2] = 3; exp[..., 3] = 2
    torch.testing.assert_close(feats.grad, exp)

    f = torch.randn(2, 5, 100, device="cuda", requires_grad=True)
    gidx = torch.randint(0, 100, (2, 10, 4), device="cuda", dtype=torch.int32)
    pu.grouping_operation(f, gidx).square().sum().backward()
    ref = torch.zeros_like(f)
    vals = torch.gather(f.detach()[:, :, None].expand(-1, -1, 10, -1), 3, gidx.long()[:, None].expand(-1, 5, -1, -1))
    ref.scatter_add_(2, gidx.long().reshape(2, 1, 40).expand(-1, 5, -1), (2 * vals).reshape(2, 5, 40))
    torch.testing.assert_close(f.grad, ref, atol=1e-5, rtol=1e-5)

    sa = PointnetSAModuleVotes(radius=0.2, nsample=64, npoint=256, mlp=[0, 64, 128, 256], normalize_xyz=True).cuda()
    pc = cu(synthetic.point_clouds(2, 4000, seed=1))
    new_xyz, new_feats, inds = sa(pc)
    assert new_xyz.shape == (2, 256, 3) and new_feats.shape == (2, 256, 256) and inds.dtype == torch.int32
    new_feats.sum().backward()
    assert sa.mlp_module.layer0.conv.weight.grad is not None
