"""Synchronised BatchNorm (ops.set_bn_sync / TrainStep(sync_bn=True)) and the bias column sum of csrc/sa_mlp_kernels.cu
against float64.

1. The kernels through ctypes, in one process: coda_bn_rows_sums, coda_bn_partials_sums on the partials of the fp32-A
   GEMM's statistics epilogue, coda_bn_stats_finalize_sums, and coda_rows_colsum.  With one rank the sums path must give
   the bits of the per-GPU path (both finish with the same fp64 formula); W simulated ranks add their fp64 sums on the
   device in place of the all-reduce and must give the statistics of the concatenated batch.
2. The ops and modules on three gloo ranks sharing one GPU, each with an equal slice of one batch, against fp64
   whole-batch BatchNorm (what torch's SyncBatchNorm computes): ops.bn_act_rows, the fused shared-MLP node
   (sa_mlp._SharedMLPMax) and the masked encoder's interim set-abstraction module, which runs its shared MLP module by
   module.

The sync path shares bn_stats_partial_kernel and warp_partials_sum with the per-GPU path, so it is held to the bars of
tests/test_sa_mlp_edges_gpu.py (and of tests/test_step_glue_edges_gpu.py for ops.bn_act_rows).
tests/test_sa_mlp_paths_cpu.py checks that the case lists below reach every width and both sides of every grid-stride
loop of the sums and column-sum kernels."""
import copy
import ctypes
import datetime
import os
import socket

import pytest
import torch

import gemm_instances as G
import sa_mlp_paths as P
import test_sa_mlp_edges_gpu as E

pytestmark = pytest.mark.gpu

_i, _ll, _f = ctypes.c_int, ctypes.c_longlong, ctypes.c_float
_call, _p, _ok, _rel, _sum_rel = E._call, E._p, E._ok, E._rel, E._sum_rel
EPS, MOMENTUM = E.EPS, E.MOMENTUM


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _pad64(c):
    return (c + 63) // 64 * 64


def _sums64(y):
    y64 = y.double()
    return y64, torch.cat((y64.sum(0), (y64 * y64).sum(0)))


def _rows_sums(y):
    rows, c = y.shape
    sums = torch.full((2 * c,), float("nan"), dtype=torch.float64, device="cuda")
    _call("coda_bn_rows_sums", _ll(rows), _i(c), _p(y), _p(sums), _p(E._scratch(c)))
    return sums


def _partials_sums(part):
    nblocks, _, c = part.shape
    sums = torch.full((2 * c,), float("nan"), dtype=torch.float64, device="cuda")
    _call("coda_bn_partials_sums", _i(nblocks), _i(c), _p(part), _p(sums))
    return sums


def _finalize_sums(rows, c, sums, rm=None, rv=None, gamma=None, beta=None, guard=0):
    """-> mean, invstd (each c + guard floats, NaN-filled) and scale / shift (pad64(c) + guard, NaN-filled) or None"""
    mean = torch.full((c + guard,), float("nan"), device="cuda")
    invstd = torch.full((c + guard,), float("nan"), device="cuda")
    scale = shift = None
    if gamma is not None:
        scale = torch.full((_pad64(c) + guard,), float("nan"), device="cuda")
        shift = torch.full((_pad64(c) + guard,), float("nan"), device="cuda")
    _call("coda_bn_stats_finalize_sums", _ll(rows), _i(c), _p(sums), _f(EPS), _f(MOMENTUM), _p(rm), _p(rv), _p(gamma),
          _p(beta), _p(mean), _p(invstd), _p(scale), _p(shift))
    return mean, invstd, scale, shift


def _running(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(c, device="cuda", generator=g) * 0.1, torch.rand(c, device="cuda", generator=g) + 0.5


def _gamma_beta(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(c, device="cuda", generator=g) + 0.5, torch.randn(c, device="cuda", generator=g) * 0.3


# ====================================================================== coda_bn_rows_sums

STEP_ROWS = 8 * 2048 * 64        # the step's pre-encoder: 8 scenes x 2048 seeds x 64 neighbours
SUMS_CASES = E.ROW_CASES + [(c, STEP_ROWS) for c in (64, 128, 256)]


def _check_sums(sums, y64, what):
    c = y64.shape[1]
    _ok(_sum_rel(sums[:c], y64), E.STATS_BAR, f"{what} column sums")
    _ok(_rel(sums[c:], (y64 * y64).sum(0)), E.STATS_BAR, f"{what} column sums of squares")


@pytest.mark.parametrize("c,rows", SUMS_CASES)
def test_bn_rows_sums_vs_fp64(c, rows):
    """fp64 column sums and sums of squares of a pass over y, on the scale of the summed magnitudes"""
    y = E._rows_with_offsets(rows, c, rows + c)
    sums = _rows_sums(y)
    y64 = y.double()
    del y
    _check_sums(sums, y64, "rows")


@pytest.mark.parametrize("ratio", E.OFFSET_RATIOS)
def test_bn_rows_sums_with_offset_means(ratio):
    """1 M rows at 256 channels whose means lie `ratio` standard deviations from zero, through rows_sums and
    finalize_sums: the per-GPU path's bars, and its bits"""
    rows, c = 1 << 20, 256
    torch.manual_seed(ratio)
    sigma = torch.rand(c, device="cuda") + 0.5
    sign = torch.where(torch.rand(c, device="cuda") < 0.5, -1.0, 1.0)
    y = torch.randn(rows, c, device="cuda") * sigma + sign * ratio * sigma
    mean, invstd, _, _ = _finalize_sums(rows, c, _rows_sums(y))
    mean1, invstd1 = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_rows_stats", _ll(rows), _i(c), _p(y), _f(EPS), _f(MOMENTUM), _p(None), _p(None), _p(mean1),
          _p(invstd1), _p(E._scratch(c)))
    assert torch.equal(mean, mean1) and torch.equal(invstd, invstd1)
    m64, v64 = E._stats64(y)
    del y
    _ok(float(((mean.double() - m64).abs() / (v64 + m64 * m64).sqrt()).max()), E.STATS_BAR, "mean")
    _ok(_rel(invstd, 1.0 / torch.sqrt(v64 + EPS)), E.OFFSET_BAR[ratio], f"invstd at {ratio} std")


# ====================================================================== coda_bn_partials_sums

# (nsplit, m, n, k, mode): the fp32-A GEMM instances sa_mlp takes with statistics; tests/test_sa_mlp_paths_cpu.py checks
# that they reach a plain first layer, the AFFINE_RELU layers and the B-resident grid, and both sides of it
PARTIAL_CASES = [
    (3, 8449, 128, 64, G.A32_PLAIN),                # GEMM first layer, one row past the last full tile
    (3, 4097, 64, 64, G.A32_PLAIN),                 # 64 wide
    (3, 9001, 256, 128, G.A32_AFFINE_RELU),         # a later layer, 256 wide
    (3, 70001, 64, 64, G.A32_AFFINE_RELU),          # B-resident grid, ragged m
    (3, STEP_ROWS, 128, 64, G.A32_AFFINE_RELU),     # the step's pre-encoder layers 2 and 3: B-resident
    (3, STEP_ROWS, 256, 128, G.A32_AFFINE_RELU),
]


def _gemm_partials(ns, m, n, k, mode, seed):
    """(y, partials) of one gemm_a32 call with the statistics epilogue, as sa_mlp._SharedMLPMax runs it"""
    from coda_neurips2023_b200 import ops

    torch.manual_seed(seed)
    a = torch.randn(m, k, device="cuda")
    w = torch.randn(n, k, device="cuda") / k ** 0.5
    kw = {}
    if mode == G.A32_AFFINE_RELU:
        kw = dict(scale=torch.rand(_pad64(k), device="cuda") + 0.5, shift=torch.rand(_pad64(k), device="cuda") - 0.3)
    return ops.gemm_a32(a, ops.pack_split(w, n, k, k, 1, ns), n, mode=mode, want_stats=True, nsplit=ns, **kw)


@pytest.mark.parametrize("ns,m,n,k,mode", PARTIAL_CASES)
def test_bn_partials_sums_vs_fp64_of_the_gemm_output(ns, m, n, k, mode):
    """fp64 sums of the GEMM epilogue's partials against fp64 sums of that GEMM's own output; partials_sums +
    finalize_sums give the bits of coda_bn_stats_finalize, running buffers included"""
    y, part = _gemm_partials(ns, m, n, k, mode, m + n + k)
    sums = _partials_sums(part)
    rm0, rv0 = _running(n, m)
    gamma, beta = _gamma_beta(n, m + 1)
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd, scale, shift = _finalize_sums(m, n, sums, rm, rv, gamma, beta)
    rm1, rv1 = rm0.clone(), rv0.clone()
    mean1, invstd1 = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    scale1, shift1 = torch.full((_pad64(n),), float("nan"), device="cuda"), torch.full((_pad64(n),), float("nan"),
                                                                                         device="cuda")
    _call("coda_bn_stats_finalize", _i(part.shape[0]), _ll(m), _i(n), _p(part), _f(EPS), _f(MOMENTUM), _p(rm1), _p(rv1),
          _p(gamma), _p(beta), _p(mean1), _p(invstd1), _p(scale1), _p(shift1))
    for got, want, what in ((mean, mean1, "mean"), (invstd, invstd1, "invstd"), (scale, scale1, "scale"),
                            (shift, shift1, "shift"), (rm, rm1, "running_mean"), (rv, rv1, "running_var")):
        assert torch.equal(got, want), f"{what}: the sums path drifts from coda_bn_stats_finalize"
    y64 = y.double()
    del y
    _check_sums(sums, y64, "GEMM partials")
    E._check_stats(m, n, y64, mean, invstd, rm0, rv0, rm, rv, gamma, beta, scale, shift)


# ====================================================================== coda_bn_stats_finalize_sums

GUARD = 64


@pytest.mark.parametrize("c,rows", E.FINALIZE_CASES)
def test_bn_stats_finalize_sums_vs_fp64(c, rows):
    """mean, invstd, running buffers (unbiased over the count passed), scale / shift from exact fp64 sums; the entries
    from c up to pad64(c) come back as zeros; without scale / shift nothing past the c outputs is written"""
    y = E._rows_with_offsets(rows, c, 3 * rows + c)
    y64, sums = _sums64(y)
    rm0, rv0 = _running(c, rows)
    gamma, beta = _gamma_beta(c, rows + 1)
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd, scale, shift = _finalize_sums(rows, c, sums, rm, rv, gamma, beta, GUARD)
    E._check_stats(rows, c, y64, mean[:c], invstd[:c], rm0, rv0, rm, rv, gamma, beta, scale, shift)
    for t, n, what in ((mean, c, "mean"), (invstd, c, "invstd"), (scale, _pad64(c), "scale"),
                       (shift, _pad64(c), "shift")):
        assert t[n:].isnan().all(), f"{what}: written past its end"

    # no scale / shift, no running buffers: the c outputs and nothing else
    mean2, invstd2, _, _ = _finalize_sums(rows, c, sums, guard=GUARD)
    assert torch.equal(mean2[:c], mean[:c]) and torch.equal(invstd2[:c], invstd[:c])
    assert mean2[c:].isnan().all() and invstd2[c:].isnan().all()


def test_bn_stats_finalize_sums_at_two_rows_and_zero_variance():
    """2 rows (unbiased factor 2) and a constant column (variance 0, clamped, invstd = 1 / sqrt(eps))"""
    c = 64
    y = torch.randn(2, c, device="cuda")
    y[:, 5] = 3.25
    y64, sums = _sums64(y)
    rm0, rv0 = _running(c, 2)
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd, _, _ = _finalize_sums(2, c, sums, rm, rv)
    E._check_stats(2, c, y64, mean, invstd, rm0, rv0, rm, rv)
    assert float(mean[5]) == 3.25 and float(invstd[5]) == pytest.approx(EPS ** -0.5, rel=1e-6)


# ====================================================================== one rank: the bits of the per-GPU path

@pytest.mark.parametrize("c,rows", E.ROW_CASES)
def test_rows_sums_path_gives_the_per_gpu_bits_with_one_rank(c, rows):
    """rows_sums + finalize_sums against coda_bn_rows_stats_affine and coda_bn_rows_stats: mean, invstd, scale,
    shift and running buffers, bit for bit"""
    y = E._rows_with_offsets(rows, c, rows + 5 * c)
    sums = _rows_sums(y)
    rm0, rv0 = _running(c, rows + c)
    gamma, beta = _gamma_beta(c, rows)
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd, scale, shift = _finalize_sums(rows, c, sums, rm, rv, gamma, beta)

    rm1, rv1 = rm0.clone(), rv0.clone()
    mean1, invstd1 = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    scale1, shift1 = torch.empty(_pad64(c), device="cuda"), torch.empty(_pad64(c), device="cuda")
    _call("coda_bn_rows_stats_affine", _ll(rows), _i(c), _p(y), _f(EPS), _f(MOMENTUM), _p(rm1), _p(rv1), _p(gamma),
          _p(beta), _p(mean1), _p(invstd1), _p(scale1), _p(shift1), _p(E._scratch(c)))
    rm2, rv2 = rm0.clone(), rv0.clone()
    mean2, invstd2 = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_rows_stats", _ll(rows), _i(c), _p(y), _f(EPS), _f(MOMENTUM), _p(rm2), _p(rv2), _p(mean2),
          _p(invstd2), _p(E._scratch(c)))
    for got, a, b, what in ((mean, mean1, mean2, "mean"), (invstd, invstd1, invstd2, "invstd"),
                            (rm, rm1, rm2, "running_mean"), (rv, rv1, rv2, "running_var")):
        assert torch.equal(got, a) and torch.equal(got, b), f"{what}: the sums path drifts from the per-GPU path"
    assert torch.equal(scale, scale1) and torch.equal(shift, shift1)


# ====================================================================== W simulated ranks

def _rank_cases():
    out = [(w, "rows", c, P.slots(c) * 37 + 1) for w in (2, 3, 8) for c in P.WIDTHS]
    out += [(w, "gemm", 128, 3001) for w in (2, 3, 8)]
    return out


RANK_CASES = _rank_cases()


@pytest.mark.parametrize("world,source,c,rows", RANK_CASES)
def test_simulated_ranks_give_the_statistics_of_the_concatenated_batch(world, source, c, rows):
    """each of `world` equal row slices takes its own sums (a pass over its rows, or its GEMM's partials), the slices'
    sums are added on the device in place of the all-reduce, and finalize_sums over world * rows must give the
    statistics and running-buffer update of the whole batch"""
    if source == "rows":
        y = E._rows_with_offsets(world * rows, c, world * 1000 + c)
        per_rank = [_rows_sums(y[r * rows:(r + 1) * rows]) for r in range(world)]
    else:
        outs = [_gemm_partials(3, rows, c, 64, G.A32_PLAIN, 17 * r + world) for r in range(world)]
        y = torch.cat([o[0] for o in outs])
        per_rank = [_partials_sums(o[1]) for o in outs]
    total = per_rank[0].clone()
    for s in per_rank[1:]:
        total += s
    rm0, rv0 = _running(c, world + c)
    gamma, beta = _gamma_beta(c, world)
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd, scale, shift = _finalize_sums(world * rows, c, total, rm, rv, gamma, beta)
    E._check_stats(world * rows, c, y, mean, invstd, rm0, rv0, rm, rv, gamma, beta, scale, shift)


# ====================================================================== coda_rows_colsum / ops.colsum

# column sums on the scale of the summed magnitudes, as the backward reductions; measured on an H100 80GB HBM3:
# 6.0e-8 (kernel and tensor reduction), 6.0e-9 (ops.linear's bias gradient)
COLSUM_BAR = E.REDUCE_BAR
COLSUM_CASES = [(c, rows) for c in P.WIDTHS
                for rows in (2, P.COLSUM_BLOCKS * P.slots(c), P.COLSUM_BLOCKS * P.slots(c) + 1, 1 << 20)]


@pytest.mark.parametrize("c,rows", COLSUM_CASES)
def test_rows_colsum_vs_fp64(c, rows):
    """2 rows, a full 132-block grid with one row per slot, one row more (a second grid-stride step for one slot),
    and 1 M rows"""
    torch.manual_seed(rows + c)
    x = torch.randn(rows, c, device="cuda")
    out = torch.full((c + GUARD,), float("nan"), device="cuda")
    scratch = torch.empty(P.COLSUM_BLOCKS * c, device="cuda")
    _call("coda_rows_colsum", _ll(rows), _i(c), _p(x), _p(out), _p(scratch))
    assert out[c:].isnan().all(), "written past the c outputs"
    _ok(_sum_rel(out[:c], x.double()), COLSUM_BAR, "colsum")
    # ops.colsum runs the same kernel
    from coda_neurips2023_b200 import ops

    assert torch.equal(ops.colsum(x), out[:c])


@pytest.mark.parametrize("c,strided", [(2, False), (3, False), (12, False), (64, True)])
def test_colsum_tensor_reduction_for_what_the_kernel_does_not_cover(c, strided, monkeypatch):
    """widths the row kernel does not take (the 2- / 3- / 12-wide heads) and a non-contiguous input take the plain
    tensor reduction, with and without `out`"""
    from coda_neurips2023_b200 import _lib, ops

    class _NoKernel:
        def __getattr__(self, name):
            assert name != "coda_rows_colsum", "the kernel was called"
            return getattr(_lib.lib(), name)

    torch.manual_seed(c)
    base = torch.randn(3001, 2 * c, device="cuda")
    x = base[:, ::2] if strided else base[:, :c].contiguous()
    assert x.is_contiguous() != strided
    monkeypatch.setattr(ops, "lib", lambda: _NoKernel())
    got = ops.colsum(x)
    out = torch.full((c,), float("nan"), device="cuda")
    got2 = ops.colsum(x, out=out)
    assert got2.data_ptr() == out.data_ptr() and torch.equal(got, got2)
    _ok(_sum_rel(got, x.double()), COLSUM_BAR, "colsum")


@pytest.mark.parametrize("relu", [False, True])
def test_linear_bias_gradient_through_the_colsum_kernel(relu, monkeypatch):
    """ops.linear with k = 259 (the masked encoder's interim MLP input: 256 features + 3 xyz): the fused column sum
    of gemm_tn32 declines and the bias gradient comes from coda_rows_colsum; against fp64 autograd, with the ReLU
    routed by the kernel's own output sign"""
    from coda_neurips2023_b200 import ops

    m, k, n = 8449, 259, 256
    torch.manual_seed(m + int(relu))
    x = torch.randn(m, k, device="cuda")
    w = (torch.randn(n, k, device="cuda") / k ** 0.5).requires_grad_(True)
    b = (torch.randn(n, device="cuda") * 0.1).requires_grad_(True)
    gout = torch.randn(m, n, device="cuda")
    calls = []
    colsum = ops.colsum

    def spy(t, out=None):
        calls.append(t.shape)
        return colsum(t, out=out)

    monkeypatch.setattr(ops, "colsum", spy)
    y = ops.linear(x, w, b, relu=relu)
    y.backward(gout)
    assert calls == [(m, n)], "the bias gradient did not come from ops.colsum"

    x64, w64 = x.double(), w.detach().double()
    b64 = b.detach().double().requires_grad_(True)
    z = x64 @ w64.t() + b64
    if relu:
        z = z * (y.detach() > 0)
    (z * gout.double()).sum().backward()
    terms = gout.double() * (y.detach() > 0) if relu else gout.double()
    # on the scale of the summed magnitudes (sums of random signs cancel)
    err = (b.grad.double() - b64.grad).abs() / terms.abs().sum(0)
    _ok(float(err.max()), COLSUM_BAR, "bias grad")


# ====================================================================== gloo ranks sharing one GPU

WORLD = 3
# bars of tests/test_step_glue_edges_gpu.py::test_bn_act_rows_vs_fp64; measured here on an H100 80GB HBM3: out 1.2e-7,
# dx 1.2e-7, dgamma 2.0e-7, dbeta 7.9e-8, running_var 6.4e-8
ACT_OUT_BAR, ACT_DY_BAR, ACT_DGAMMA_BAR, ACT_DBETA_BAR = 1.8e-5, 2e-5, 2e-5, 1.5e-6
ACT_RM_BAR, ACT_RV_BAR = 1e-6, 1e-5
# (c, rows per rank, relu)
ACT_CASES = [(64, 3001, False), (64, 3001, True), (256, 1001, False), (256, 1001, True)]
# (spec, scenes per rank, npoint, group, x_grad): the pre-encoder (small-K first layer, statistics from rows_sums) and
# a GEMM first layer (statistics from the GEMM partials) with an input gradient
NODE_RANK_CASES = [([3, 64, 128, 256], 2, 151, 64, False), ([64, 128, 256], 1, 111, 32, True)]
# the masked encoder's interim PointnetSAModuleVotes (models/model_3detr.py: build_encoder) at 2048 pre-encoder points
ENC_NPOINT, ENC_NSAMPLE, ENC_RADIUS, ENC_DIM, ENC_POINTS = 1024, 32, 0.4, 256, 2048


def _act_inputs(c, rows, relu):
    """(y, gout, bn) of the whole batch, the same in every process; with the ReLU, the y whose whole-batch fp64
    BatchNorm output lies within 1e-3 of the edge move 2e-3 further out, so that fp32 and fp64 agree on the mask"""
    g = torch.Generator().manual_seed(c * 10 + int(relu))
    n = WORLD * rows
    y = torch.randn(n, c, generator=g) * (torch.rand(c, generator=g) + 0.5) + torch.randn(c, generator=g)
    gout = torch.randn(n, c, generator=g)
    bn = torch.nn.BatchNorm1d(c)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g) * 0.3)
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    if relu:
        y64 = y.double()
        mean, invstd = y64.mean(0), 1.0 / torch.sqrt(y64.var(0, unbiased=False) + bn.eps)
        E._off_relu_edge(y, mean, invstd, bn.weight.detach(), bn.bias.detach())
    return y, gout, bn


def _node_inputs(spec, b, npoint, group):
    g = torch.Generator().manual_seed(sum(spec) + npoint)
    x = torch.randn(WORLD * b * npoint * group, spec[0], generator=g)
    gout = torch.randn(WORLD * b * npoint, spec[-1], generator=g)
    return x, gout


def _encoder_module():
    from coda_neurips2023_b200.pointnet2.pointnet2_modules import PointnetSAModuleVotes

    torch.manual_seed(930)
    mod = PointnetSAModuleVotes(radius=ENC_RADIUS, nsample=ENC_NSAMPLE, npoint=ENC_NPOINT,
                                mlp=[ENC_DIM, 256, 256, ENC_DIM], normalize_xyz=True)
    g = torch.Generator().manual_seed(931)
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.3)
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.8)
    return mod.cuda().train()


def _encoder_inputs():
    from coda_neurips2023_b200 import synthetic

    xyz = torch.from_numpy(synthetic.point_clouds(WORLD, ENC_POINTS, seed=29))
    feats = torch.randn(WORLD, ENC_DIM, ENC_POINTS, generator=torch.Generator().manual_seed(29))
    return xyz, feats


def _rank_worker(rank, world, port, outdir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    from coda_neurips2023_b200 import ops

    torch.cuda.set_device(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    ops.set_bn_sync(True)
    assert ops.bn_sync_world() == world
    res = {}
    for c, rows, relu in ACT_CASES:
        y, gout, bn = _act_inputs(c, rows, relu)
        bn = bn.cuda().train()
        sl = slice(rank * rows, (rank + 1) * rows)
        h = y[sl].cuda().requires_grad_(True)
        out = ops.bn_act_rows(h, bn, relu, 0.0, True)
        out.backward(gout[sl].cuda())
        res[("act", c, relu)] = dict(out=out.detach().cpu(), dx=h.grad.cpu(), dgamma=bn.weight.grad.cpu(),
                                     dbeta=bn.bias.grad.cpu(), buffers={k: v.cpu() for k, v in bn.state_dict().items()
                                                                        if k.startswith(("running", "num_"))})
    for spec, b, npoint, group, x_grad in NODE_RANK_CASES:
        mlp = E._mlp(spec, sum(spec) + npoint)
        x, gout = _node_inputs(spec, b, npoint, group)
        n, ng = b * npoint * group, b * npoint
        xr = x[rank * n:(rank + 1) * n].cuda().requires_grad_(x_grad)
        pooled, argmax = E._node(mlp, xr, group)
        pooled.backward(gout[rank * ng:(rank + 1) * ng].cuda())
        res[("node", tuple(spec))] = dict(pooled=pooled.detach().cpu(), argmax=argmax.cpu(),
                                          dx=xr.grad.cpu() if x_grad else None,
                                          grads={k: p.grad.cpu() for k, p in mlp.named_parameters()},
                                          buffers={k: v.cpu() for k, v in mlp.named_buffers()})
    mod = _encoder_module()
    xyz, feats = _encoder_inputs()
    _, new_feats, _ = mod(xyz[rank:rank + 1].cuda(), feats[rank:rank + 1].cuda().requires_grad_(True))
    res["encoder"] = dict(pooled=new_feats.detach().cpu(),
                          buffers={k: v.cpu() for k, v in mod.mlp_module.named_buffers()})
    ops.set_bn_sync(False)
    torch.save(res, os.path.join(outdir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture(scope="module")
def ranks(tmp_path_factory):
    """the results of WORLD gloo ranks on cuda:0, each with ops.set_bn_sync(True) and an equal slice of every batch"""
    import torch.multiprocessing as mp

    outdir = str(tmp_path_factory.mktemp("sync_bn"))
    mp.spawn(_rank_worker, args=(WORLD, _free_port(), outdir), nprocs=WORLD, join=True)
    return [torch.load(os.path.join(outdir, f"rank{r}.pt")) for r in range(WORLD)]


def _same_buffers(ranks, key):
    """every rank holds the same running buffers, bit for bit"""
    first = ranks[0][key]["buffers"]
    for r in range(1, WORLD):
        for name, v in first.items():
            assert torch.equal(ranks[r][key]["buffers"][name], v), f"rank {r} {name} differs from rank 0"
    return first


@pytest.mark.parametrize("c,rows,relu", ACT_CASES)
def test_bn_act_rows_on_gloo_ranks_vs_fp64_whole_batch(ranks, c, rows, relu):
    """each rank's output and dx are its slice of whole-batch BatchNorm's; the ranks' local dgamma / dbeta sum to
    the whole batch's; the running buffers are the same on every rank and are the whole batch's"""
    y, gout, bn = _act_inputs(c, rows, relu)
    key = ("act", c, relu)
    yr = y.double().cuda().requires_grad_(True)
    wr = bn.weight.detach().double().cuda().requires_grad_(True)
    br = bn.bias.detach().double().cuda().requires_grad_(True)
    rm, rv = bn.running_mean.double().cuda(), bn.running_var.double().cuda()
    ref = torch.nn.functional.batch_norm(yr, rm, rv, wr, br, True, MOMENTUM, bn.eps)
    if relu:
        ref = ref.relu()
    ref.backward(gout.double().cuda())
    out = torch.cat([ranks[r][key]["out"] for r in range(WORLD)]).cuda()
    dx = torch.cat([ranks[r][key]["dx"] for r in range(WORLD)]).cuda()
    _ok(_rel(out, ref.detach()), ACT_OUT_BAR, "out")
    _ok(_rel(dx, yr.grad), ACT_DY_BAR, "dx")
    _ok(_rel(sum(ranks[r][key]["dgamma"] for r in range(WORLD)).cuda(), wr.grad), ACT_DGAMMA_BAR, "dgamma")
    _ok(_rel(sum(ranks[r][key]["dbeta"] for r in range(WORLD)).cuda(), br.grad), ACT_DBETA_BAR, "dbeta")
    buf = _same_buffers(ranks, key)
    _ok(_rel(buf["running_mean"].cuda(), rm), ACT_RM_BAR, "running_mean")
    _ok(_rel(buf["running_var"].cuda(), rv), ACT_RV_BAR, "running_var")
    assert int(buf["num_batches_tracked"]) == 1


@pytest.mark.parametrize("spec,b,npoint,group,x_grad", NODE_RANK_CASES)
def test_shared_mlp_node_on_gloo_ranks_vs_fp64_whole_batch(ranks, spec, b, npoint, group, x_grad):
    """the fused node on each rank's slice against the fp64 node on the whole batch, routed by the ranks' arg-max:
    pooled output, input gradient, rank-summed weight / gamma / beta gradients, running buffers (NODE_* bars)"""
    key = ("node", tuple(spec))
    mlp = E._mlp(spec, sum(spec) + npoint)
    ref = copy.deepcopy(mlp).double()
    buf = _same_buffers(ranks, key)
    mlp.load_state_dict({**mlp.state_dict(), **buf})
    for name, p in mlp.named_parameters():
        p.grad = sum(ranks[r][key]["grads"][name] for r in range(WORLD)).cuda()
    x, gout = _node_inputs(spec, b, npoint, group)
    x = x.cuda().requires_grad_(x_grad)
    if x_grad:
        x.grad = torch.cat([ranks[r][key]["dx"] for r in range(WORLD)]).cuda()
    pooled = torch.cat([ranks[r][key]["pooled"] for r in range(WORLD)]).cuda().requires_grad_(True)
    argmax = torch.cat([ranks[r][key]["argmax"] for r in range(WORLD)]).cuda()
    E._check_node(mlp, ref, x, group, x_grad, argmax, pooled, gout.cuda())


def test_masked_encoder_interim_module_syncs_its_batchnorm(ranks):
    """The masked encoder's interim set-abstraction module (mlp 259 -> 256 -> 256 -> 256, which the fused node
    declines) runs its shared MLP module by module; with synchronisation on, its three BatchNorm layers must take
    the whole batch's statistics: the same running buffers on every rank, those of fp64 BatchNorm on the
    concatenated batch, and each rank's pooled output its slice of the whole batch's.

    Measured on an H100 80GB HBM3: pooled 1.6e-6 (NODE_FWD_BAR 3e-6), running_mean 9.0e-7 (NODE_BUF_BAR 1.5e-6).  The
    margin is below the node's 3x: this path runs three GEMMs on packed operands (k = 259 is not a multiple of 4) and
    BatchNorm between them, not the fused node's prologues."""
    from coda_neurips2023_b200.pointnet2 import pointnet2_utils

    mod = _encoder_module()
    ref = copy.deepcopy(mod.mlp_module).double()
    xyz, feats = _encoder_inputs()
    xyz, feats = xyz.cuda(), feats.cuda()
    inds = pointnet2_utils.furthest_point_sample(xyz, ENC_NPOINT)
    new_xyz = pointnet2_utils.gather_operation(xyz.transpose(1, 2).contiguous(), inds).transpose(1, 2).contiguous()
    grouped, _ = mod.grouper(xyz, new_xyz, feats)                        # (W, 259, npoint, nsample)
    rows = grouped.permute(0, 2, 3, 1).reshape(-1, grouped.shape[1])
    with torch.no_grad():
        f64 = E._features64(ref, rows.double())
    exp = f64.view(WORLD, ENC_NPOINT, ENC_NSAMPLE, -1).amax(2)          # (W, npoint, 256)
    got = torch.cat([ranks[r]["encoder"]["pooled"] for r in range(WORLD)]).cuda().permute(0, 2, 1)
    _ok(float((got.double() - exp).abs().max() / exp.abs().max()), E.NODE_FWD_BAR, "encoder pooled")
    buf = _same_buffers(ranks, "encoder")
    for name, v in ref.named_buffers():
        if v.dtype.is_floating_point:
            _ok(_rel(buf[name].cuda(), v), E.NODE_BUF_BAR, f"encoder {name}")
        else:
            assert torch.equal(buf[name].cuda(), v), name
