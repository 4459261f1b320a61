"""The fp32-A wgmma GEMM with in-kernel prologues (include/coda_gemm.h, coda_gemm_a32) against fp64 references:
plain, BatchNorm+ReLU prologue, the two BatchNorm-backward prologues, K-major and MN-major weights, ragged m / n / k,
and the column-statistics epilogue."""
import numpy as np
import pytest
import torch

from coda_neurips2023_b200.ops import (A32_AFFINE_RELU as AFFINE_RELU, A32_BN_BWD as BN_BWD,
                                       A32_BN_BWD_POOLED as POOLED, A32_BN_BWD_POOLED_PRE as POOLED_PRE,
                                       A32_PLAIN as PLAIN)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


def _planes(w, ns):
    from coda_neurips2023_b200 import ops

    n, k = w.shape
    return ops.pack_split(w, n, k, k, 1, ns)


def _rel(got, exp):
    return float((got.double() - exp).abs().max() / exp.abs().max())


@pytest.mark.parametrize("m,n,k,ns", [(4096, 256, 128, 3), (1000, 128, 64, 3), (333, 48, 200, 3), (16384, 512, 512, 3),
                                       (2048, 12, 512, 3), (5000, 192, 256, 2), (128, 64, 64, 2), (70001, 128, 64, 3)])
def test_plain_matches_fp64(m, n, k, ns):
    from coda_neurips2023_b200 import ops

    torch.manual_seed(m + n + k)
    a = torch.randn(m, k, device="cuda")
    w = torch.randn(n, k, device="cuda") / k ** 0.5
    bias = torch.randn(n, device="cuda")
    got = ops.gemm_a32(a, _planes(w, ns), n, bias=bias, relu=True)
    exp = torch.relu(a.double() @ w.double().t() + bias.double())
    assert _rel(got, exp) < (6e-6 if ns == 3 else 6e-5)


def test_strided_a_and_mn_major_weight():
    """dX = dY W: A is a column slice of a wider matrix, B are the FORWARD planes of W (rows = contraction)."""
    from coda_neurips2023_b200 import ops

    torch.manual_seed(0)
    wide = torch.randn(3000, 768, device="cuda")
    dy = wide[:, 256:512]                       # (3000, 256), row stride 768
    w = torch.randn(256, 192, device="cuda") / 16       # forward weight (n_out = 256, k_in = 192)
    planes = _planes(w, 3)                              # (3, 1, 256, 192)
    got = ops.gemm_a32(dy, planes, 192, b_mn=True, nsplit=2)
    assert _rel(got, dy.double() @ w.double()) < 4e-5
    got3 = ops.gemm_a32(dy, planes, 192, b_mn=True, nsplit=3)
    assert _rel(got3, dy.double() @ w.double()) < 6e-6


def test_affine_relu_prologue_and_stats_epilogue():
    from coda_neurips2023_b200 import ops

    torch.manual_seed(1)
    m, k, n = 20000, 128, 256
    y = torch.randn(m, k, device="cuda") * 2 + 0.5
    scale = torch.rand(k, device="cuda") + 0.5
    shift = torch.randn(k, device="cuda") * 0.3
    w = torch.randn(n, k, device="cuda") / k ** 0.5
    got, part = ops.gemm_a32(y, _planes(w, 3), n, mode=ops.A32_AFFINE_RELU, scale=scale, shift=shift, want_stats=True)
    a = torch.relu(y.double() * scale.double() + shift.double())
    exp = a @ w.double().t()
    assert _rel(got, exp) < 6e-6
    s = part.double().sum(0)
    # the epilogue sums exactly the values it stores (fp32 partial sums per 32-row group, fp64 across groups)
    g = got.double()
    assert torch.allclose(s[0], g.sum(0), rtol=1e-6, atol=2e-3)
    assert torch.allclose(s[1], (g * g).sum(0), rtol=1e-6, atol=2e-3)
    assert torch.allclose(s[0], exp.sum(0), rtol=1e-5, atol=0.1)


def test_bn_backward_prologues():
    from coda_neurips2023_b200 import ops

    torch.manual_seed(2)
    m, k, n, group = 64 * 300, 256, 128, 64
    y = torch.randn(m, k, device="cuda")
    d = torch.randn(m, k, device="cuda")
    scale = torch.rand(k, device="cuda") + 0.5
    shift = torch.randn(k, device="cuda") * 0.3
    alpha = torch.randn(k, device="cuda") * 0.01
    beta = torch.randn(k, device="cuda") * 0.01
    w = torch.randn(k, n, device="cuda") / k ** 0.5      # forward weight (k_out = contraction here, n = its input dim)
    planes = _planes(w, 3)
    z = y.double() * scale.double() + shift.double()
    dy = (z > 0) * scale.double() * d.double() + y.double() * alpha.double() + beta.double()
    got = ops.gemm_a32(y, planes, n, mode=ops.A32_BN_BWD, scale=scale, shift=shift, alpha=alpha, beta=beta, a2=d,
                       b_mn=True, nsplit=2)
    assert _rel(got, dy @ w.double()) < 6e-5
    # pooled form
    dp = torch.randn(m // group, k, device="cuda")
    arg = torch.randint(0, group, (m // group, k), device="cuda", dtype=torch.uint8)
    dfull = torch.zeros(m // group, group, k, device="cuda", dtype=torch.float64)
    dfull.scatter_(1, arg.long().unsqueeze(1), dp.double().unsqueeze(1))
    dyp = (z > 0) * scale.double() * dfull.view(m, k) + y.double() * alpha.double() + beta.double()
    gotp = ops.gemm_a32(y, planes, n, mode=ops.A32_BN_BWD_POOLED, scale=scale, shift=shift, alpha=alpha, beta=beta,
                        a2=dp, argmax=arg, group=group, b_mn=True, nsplit=2)
    assert _rel(gotp, dyp @ w.double()) < 6e-5
    # pre-masked, pre-scaled pooled gradient (what the step uses): the same values, fewer prologue instructions
    zmax = torch.gather(z.view(m // group, group, k), 1, arg.long().unsqueeze(1)).squeeze(1)
    dprime = ((zmax > 0) * scale.double() * dp.double()).float()
    gotq = ops.gemm_a32(y, planes, n, mode=ops.A32_BN_BWD_POOLED_PRE, scale=scale, shift=shift, alpha=alpha, beta=beta,
                        a2=dprime, argmax=arg, group=group, b_mn=True, nsplit=2)
    assert _rel(gotq, dyp @ w.double()) < 6e-5


@pytest.mark.parametrize("rows,m,n", [(65536, 256, 128), (10000, 128, 64), (4099, 512, 512), (700, 12, 512),
                                      (131072, 64, 128)])
def test_tn32_plain_matches_fp64(rows, m, n):
    from coda_neurips2023_b200 import ops

    torch.manual_seed(rows + m)
    a = torch.randn(rows, m, device="cuda")
    b = torch.randn(rows, n, device="cuda")
    got = ops.gemm_tn32(a, b)
    exp = a.double().t() @ b.double()
    assert _rel(got, exp) < 6e-5
    # split-K over the rows: partial tiles and column sums are added in split order, the same bits on every call
    cs1, cs2 = torch.empty(m, device="cuda"), torch.empty(m, device="cuda")
    got1 = ops.gemm_tn32(a, b, colsum_out=cs1)
    assert torch.equal(got1, got)
    assert torch.equal(ops.gemm_tn32(a, b, colsum_out=cs2), got1) and torch.equal(cs1, cs2)
    torch.testing.assert_close(cs1.double(), a.double().sum(0), rtol=1e-5, atol=1e-3)


def test_tn32_bn_backward_and_forward_prologues():
    from coda_neurips2023_b200 import ops

    torch.manual_seed(5)
    rows, m, n, group = 64 * 500, 256, 128, 64
    y = torch.randn(rows, m, device="cuda")
    d = torch.randn(rows, m, device="cuda")
    sa, ta = torch.rand(m, device="cuda") + 0.5, torch.randn(m, device="cuda") * 0.3
    al, be = torch.randn(m, device="cuda") * 0.01, torch.randn(m, device="cuda") * 0.01
    yp = torch.randn(rows, n, device="cuda")
    sb, tb = torch.rand(n, device="cuda") + 0.5, torch.randn(n, device="cuda") * 0.3
    x = torch.relu(yp.double() * sb.double() + tb.double())
    z = y.double() * sa.double() + ta.double()
    dy = (z > 0) * sa.double() * d.double() + y.double() * al.double() + be.double()
    got = ops.gemm_tn32(y, yp, a_mode=ops.A32_BN_BWD, a_scale=sa, a_shift=ta, a_alpha=al, a_beta=be, a2=d,
                        b_mode=ops.A32_AFFINE_RELU, b_scale=sb, b_shift=tb)
    assert _rel(got, dy.t() @ x) < 6e-5
    dp = torch.randn(rows // group, m, device="cuda")
    arg = torch.randint(0, group, (rows // group, m), device="cuda", dtype=torch.uint8)
    dfull = torch.zeros(rows // group, group, m, device="cuda", dtype=torch.float64)
    dfull.scatter_(1, arg.long().unsqueeze(1), dp.double().unsqueeze(1))
    dyp = (z > 0) * sa.double() * dfull.view(rows, m) + y.double() * al.double() + be.double()
    gotp = ops.gemm_tn32(y, yp, a_mode=ops.A32_BN_BWD_POOLED, a_scale=sa, a_shift=ta, a_alpha=al, a_beta=be, a2=dp,
                         argmax=arg, group=group, b_mode=ops.A32_AFFINE_RELU, b_scale=sb, b_shift=tb)
    assert _rel(gotp, dyp.t() @ x) < 6e-5
    zmax = torch.gather(z.view(rows // group, group, m), 1, arg.long().unsqueeze(1)).squeeze(1)
    dprime = ((zmax > 0) * sa.double() * dp.double()).float()
    gotq = ops.gemm_tn32(y, yp, a_mode=ops.A32_BN_BWD_POOLED_PRE, a_scale=sa, a_shift=ta, a_alpha=al, a_beta=be,
                         a2=dprime, argmax=arg, group=group, b_mode=ops.A32_AFFINE_RELU, b_scale=sb, b_shift=tb)
    assert _rel(gotq, dyp.t() @ x) < 6e-5


# ---------------------------------------------------------------- every instance, tails, prologue padding, statistics

# (nsplit, m, n, k, b_mn, mode, stats, relu): tests/test_gemm_instances_cpu.py checks that these reach every instance
# coda_gemm_a32 can select (both weight layouts) and the B-resident grid.
A32_CASES = [
    (2, 1, 48, 64, False, PLAIN, False, True),           # m = 1
    (2, 8448, 128, 200, False, PLAIN, False, False),     # 66 tiles of 128 x 128: 64-wide tiles ...
    (2, 8449, 128, 200, False, AFFINE_RELU, False, True),   # ... 67: 128-wide
    (3, 64, 200, 12, False, AFFINE_RELU, False, False),  # m = 64
    (3, 9000, 192, 200, False, AFFINE_RELU, False, True),   # deep B ring
    (3, 8449, 256, 100, False, PLAIN, True, True),       # statistics, one row past the last full tile
    (2, 127, 256, 4096, True, PLAIN, False, False),      # m = 127; the K / V bank's 4096-long contraction
    (2, 4100, 512, 4096, True, PLAIN, False, False),     # ... at the bank's width
    (2, 5000, 256, 200, True, BN_BWD, False, False),
    (3, 64, 100, 12, True, BN_BWD, False, False),
    (3, 9000, 192, 200, True, AFFINE_RELU, False, False),   # <3, 128, *, MN> with the deep B ring ...
    (3, 9000, 192, 12, True, PLAIN, False, True),        # ... and without (short k)
    (3, 9000, 192, 200, True, BN_BWD, False, False),     # ... and without (two-input prologue)
    (3, 70001, 48, 64, False, AFFINE_RELU, True, True),  # B-resident grid with statistics, ragged m
]


def _per_k(values, pad_value):
    """per-k coefficient vector padded to a multiple of 64; the padding holds `pad_value`, or random values if None"""
    k = values.numel()
    kpad = (k + 63) // 64 * 64
    v = torch.full((kpad,), float(pad_value), device="cuda") if pad_value is not None else \
        torch.randn(kpad, device="cuda") * 3
    v[:k] = values
    return v


@pytest.mark.parametrize("ns,m,n,k,b_mn,mode,stats,relu", A32_CASES)
def test_a32_instances_and_edges_vs_fp64(ns, m, n, k, b_mn, mode, stats, relu):
    from coda_neurips2023_b200 import ops

    torch.manual_seed(m + n + k)
    a = torch.randn(m, k, device="cuda")
    d = torch.randn(m, k, device="cuda")
    # B: K-major planes of W (n, k), or the forward planes of W^T (k rows, n wide) read MN-major
    w = torch.randn(k, n, device="cuda") / k ** 0.5 if b_mn else torch.randn(n, k, device="cuda") / k ** 0.5
    wt = w.double() if b_mn else w.double().t()        # (k, n)
    planes = _planes(w, 3)
    bias = torch.randn(n, device="cuda")
    coef = {}
    if mode != PLAIN:
        coef = dict(scale=torch.rand(k, device="cuda") + 0.5, shift=torch.rand(k, device="cuda") * 0.6 - 0.3)
    if mode == BN_BWD:
        coef.update(alpha=torch.rand(k, device="cuda") * 0.1 - 0.05, beta=torch.rand(k, device="cuda") * 0.1 - 0.05)

    def run(pad_value):
        kw = {key: _per_k(v, pad_value) for key, v in coef.items()}
        if mode == BN_BWD:
            kw["a2"] = d
        return ops.gemm_a32(a, planes, n, mode=mode, b_mn=b_mn, bias=bias, relu=relu, want_stats=stats, nsplit=ns, **kw)

    got = run(0.0)
    # the prologue of the padding columns past k must not reach C, whatever finite values the vectors hold there
    got2 = run(None)
    coef = {key: v.double() for key, v in coef.items()}
    if stats:
        (got, part), (got2, part2) = got, got2
        assert torch.equal(part, part2)
    assert torch.equal(got, got2)
    x = a.double()
    if mode == AFFINE_RELU:
        x = torch.relu(x * coef["scale"] + coef["shift"])
    elif mode == BN_BWD:
        z = x * coef["scale"] + coef["shift"]
        x = (z > 0) * coef["scale"] * d.double() + x * coef["alpha"] + coef["beta"]
    exp = x @ wt + bias.double()
    if relu:
        exp = exp.relu()
    assert _rel(got, exp) < (6e-6 if ns == 3 else 6e-5)
    if stats:
        # rows >= m are padding: their bias (+ ReLU) values must not be counted
        s, g = part.double().sum(0), got.double()
        assert torch.allclose(s[0], g.sum(0), rtol=1e-6, atol=2e-3)
        assert torch.allclose(s[1], (g * g).sum(0), rtol=1e-6, atol=2e-3)


# (rows, m, n, a_mode, b_affine, sliced, group): tests/test_gemm_instances_cpu.py checks that these reach both tile
# widths, split-K and not, and a split count that leaves trailing splits without a slab
TN32_CASES = [
    (1, 128, 64, PLAIN, False, False, 0),
    (1, 64, 128, BN_BWD, True, True, 0),
    (31, 64, 128, BN_BWD, True, True, 0),
    (31, 128, 48, PLAIN, False, True, 0),
    (33, 256, 64, BN_BWD, False, False, 0),
    (33, 192, 132, PLAIN, True, False, 0),
    (20001, 256, 128, BN_BWD, True, True, 0),           # rows % 32 = 1 on the split-K path
    (20001, 128, 64, PLAIN, False, True, 0),
    (16960, 128, 64, PLAIN, False, False, 0),           # 132 splits of 5 slabs over 530: 26 splits read nothing
    (2000, 1536, 1408, PLAIN, False, False, 0),         # 132 tiles: no split, the column sums are stored directly
    (4096, 512, 512, PLAIN, False, True, 0),            # the K / V bank's dW: 512-wide slices of a 4096-wide gradient
    (3200, 128, 64, POOLED, True, False, 32),
    (6400, 256, 128, POOLED_PRE, False, True, 128),
    (5120, 128, 128, POOLED, False, False, 256),
]


def _tn32_case(rows, m, n, a_mode, b_affine, sliced, group, seed):
    """-> (kwargs of ops.gemm_tn32, fp64 TA(A), fp64 TB(B)); sliced: A, B and the second A input are column slices
    of wider matrices (row stride > width)"""
    from coda_neurips2023_b200 import ops

    torch.manual_seed(seed)

    def mat(r, c):
        return torch.randn(r, c + 96, device="cuda")[:, 32:32 + c] if sliced else torch.randn(r, c, device="cuda")

    def vec(c, lo, width):      # per-column coefficients, padded to 128 with non-zero values
        v = torch.randn((c + 127) // 128 * 128, device="cuda")
        v[:c] = torch.rand(c, device="cuda") * width + lo
        return v

    a, b = mat(rows, m), mat(rows, n)
    kw = {}
    ta, tb = a.double(), b.double()
    if b_affine:
        kw.update(b_mode=ops.A32_AFFINE_RELU, b_scale=vec(n, 0.5, 1.0), b_shift=vec(n, -0.3, 0.6))
        tb = torch.relu(tb * kw["b_scale"][:n].double() + kw["b_shift"][:n].double())
    if a_mode != PLAIN:
        # a non-zero beta: rows past the end must not contribute it
        kw.update(a_mode=a_mode, a_scale=vec(m, 0.5, 1.0), a_shift=vec(m, -0.3, 0.6), a_alpha=vec(m, -0.1, 0.2),
                  a_beta=vec(m, 0.2, 0.5))
        s, t, al, be = (kw[key][:m].double() for key in ("a_scale", "a_shift", "a_alpha", "a_beta"))
        z = ta * s + t
        if a_mode == BN_BWD:
            d = mat(rows, m)
            kw["a2"] = d
            ta = (z > 0) * s * d.double() + ta * al + be
        else:
            dp = torch.randn(rows // group, m, device="cuda")
            arg = torch.randint(0, group, (rows // group, m), device="cuda", dtype=torch.uint8)
            if a_mode == POOLED_PRE:
                zmax = torch.gather(z.view(rows // group, group, m), 1, arg.long().unsqueeze(1)).squeeze(1)
                dp = ((zmax > 0) * s * dp.double()).float()
                mask = 1.0
            else:
                mask = z > 0
            dfull = torch.zeros(rows // group, group, m, device="cuda", dtype=torch.float64)
            dfull.scatter_(1, arg.long().unsqueeze(1), dp.double().unsqueeze(1))
            kw.update(a2=dp, argmax=arg, group=group)
            scaled = s * dfull.view(rows, m) if a_mode == POOLED else dfull.view(rows, m)
            ta = mask * scaled + ta * al + be
    return a, b, kw, ta, tb


@pytest.mark.parametrize("rows,m,n,a_mode,b_affine,sliced,group", TN32_CASES)
def test_tn32_instances_and_edges_vs_fp64(rows, m, n, a_mode, b_affine, sliced, group):
    from coda_neurips2023_b200 import ops

    a, b, kw, ta, tb = _tn32_case(rows, m, n, a_mode, b_affine, sliced, group, rows + m + n)
    cs = torch.empty(m, device="cuda")
    got = ops.gemm_tn32(a, b, colsum_out=cs, **kw)
    assert _rel(got, ta.t() @ tb) < 6e-5
    assert _rel(cs, ta.sum(0)) < 6e-5
    cs2 = torch.full((m,), float("nan"), device="cuda")
    assert torch.equal(ops.gemm_tn32(a, b, colsum_out=cs2, **kw), got) and torch.equal(cs2, cs)


def test_tn32_same_bits_after_a_larger_launch():
    """C and the column sums of a split-K launch whose last splits are empty, then the same call after a larger
    launch has left its partial tiles and column sums in the shared scratch"""
    from coda_neurips2023_b200 import ops

    a, b, kw, _, _ = _tn32_case(16960, 128, 64, BN_BWD, True, True, 0, 1)
    cs1, cs2 = torch.empty(128, device="cuda"), torch.empty(128, device="cuda")
    c1 = ops.gemm_tn32(a, b, colsum_out=cs1, **kw)
    big_a, big_b = torch.randn(65536, 512, device="cuda"), torch.randn(65536, 256, device="cuda")
    ops.gemm_tn32(big_a, big_b, colsum_out=torch.empty(512, device="cuda"))
    assert torch.equal(ops.gemm_tn32(a, b, colsum_out=cs2, **kw), c1) and torch.equal(cs2, cs1)
