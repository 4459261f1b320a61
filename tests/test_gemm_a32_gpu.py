"""The fp32-A wgmma GEMM with in-kernel prologues (include/coda_gemm.h, coda_gemm_a32) against fp64 references:
plain, BatchNorm+ReLU prologue, the two BatchNorm-backward prologues, K-major and MN-major weights, ragged m / n / k,
and the column-statistics epilogue."""
import numpy as np
import pytest
import torch

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
