"""The fp32-A GEMM's two consumer warpgroups issue their wgmmas of each k-block in turn (coda_gemm_a32,
csrc/gemm_a32_sm90.cu).  Whatever the interleaving, C and the column-statistics rows must have the same bits on every
call, also right after a launch of another shape, and match fp64: every instance of test_gemm_a32_gpu.py's list, plus
CTAs with one tile, an odd and an even number of tiles, the one-stage raw rings and both pooled prologues."""
import pytest
import torch

import test_gemm_a32_gpu as a32
from coda_neurips2023_b200.ops import (A32_AFFINE_RELU as AFFINE_RELU, A32_BN_BWD as BN_BWD,
                                       A32_BN_BWD_POOLED as POOLED, A32_BN_BWD_POOLED_PRE as POOLED_PRE,
                                       A32_PLAIN as PLAIN)

# (nsplit, m, n, k, b_mn, mode, stats, relu, group)
GRID_CASES = [
    (3, 2048, 512, 512, False, PLAIN, False, False, 0),          # 128 tiles: one per CTA
    (2, 25600, 128, 64, False, AFFINE_RELU, False, True, 0),     # two or one
    (3, 16384, 512, 512, False, PLAIN, False, False, 0),         # four or three
    (3, 30000, 256, 200, False, AFFINE_RELU, True, False, 0),    # statistics, four or three
    (3, 50000, 256, 128, False, AFFINE_RELU, True, False, 0),    # B-resident with statistics, six or five
    (3, 20000, 256, 256, True, BN_BWD, False, False, 0),         # one raw stage (two-input prologue), three or two
    (2, 32768, 128, 256, True, POOLED_PRE, False, False, 64),    # pooled prologues
    (3, 32768, 128, 256, True, POOLED, False, False, 256),       # ... one raw stage
]
CASES = [c + (0,) for c in a32.A32_CASES] + GRID_CASES


def _inputs(ns, m, n, k, b_mn, mode, group, seed):
    from coda_neurips2023_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)       # noqa: E731
    a = rnd(m, k)
    w = rnd(k, n) / k ** 0.5 if b_mn else rnd(n, k) / k ** 0.5
    planes = ops.pack_split(w, *w.shape, w.shape[1], 1, 3)
    kw = dict(mode=mode, b_mn=b_mn, nsplit=ns)
    kpad = (k + 63) // 64 * 64
    if mode != PLAIN:
        kw.update(scale=torch.rand(kpad, device="cuda", generator=g) + 0.5, shift=rnd(kpad) * 0.3)
    if mode in (BN_BWD, POOLED, POOLED_PRE):
        kw.update(alpha=rnd(kpad) * 0.05, beta=rnd(kpad) * 0.05)
    if mode == BN_BWD:
        kw["a2"] = rnd(m, k)
    if mode in (POOLED, POOLED_PRE):
        kw.update(a2=rnd(m // group, k), group=group,
                  argmax=torch.randint(0, group, (m // group, k), device="cuda", generator=g, dtype=torch.uint8))
    return a, w, planes, kw


@pytest.mark.gpu
@pytest.mark.parametrize("ns,m,n,k,b_mn,mode,stats,relu,group", CASES)
def test_same_bits_every_call(built_lib, ns, m, n, k, b_mn, mode, stats, relu, group):
    from coda_neurips2023_b200 import ops

    a, w, planes, kw = _inputs(ns, m, n, k, b_mn, mode, group, seed=m + n + k)
    bias = torch.randn(n, device="cuda")

    def run():
        r = ops.gemm_a32(a, planes, n, bias=bias, relu=relu, want_stats=stats, **kw)
        return r if stats else (r, None)

    c0, s0 = run()
    c1, s1 = run()
    # another shape in between: other tiles per CTA, other ring positions
    o_ns, o_m, o_n, o_k, o_mn, o_mode, *_ = GRID_CASES[2] if (m, n) != (16384, 512) else GRID_CASES[3]
    oa, _, oplanes, okw = _inputs(o_ns, o_m, o_n, o_k, o_mn, o_mode, 0, seed=1)
    ops.gemm_a32(oa, oplanes, o_n, want_stats=True, **okw)
    c2, s2 = run()
    assert torch.equal(c0, c1) and torch.equal(c0, c2)
    if stats:
        assert torch.equal(s0, s1) and torch.equal(s0, s2)
        g = c0.double()
        torch.testing.assert_close(s0.double().sum(0)[0], g.sum(0), rtol=1e-6, atol=2e-3)
        torch.testing.assert_close(s0.double().sum(0)[1], (g * g).sum(0), rtol=1e-6, atol=2e-3)
    if mode == PLAIN:
        exp = a.double() @ (w.double() if b_mn else w.double().t()) + bias.double()
        if relu:
            exp = torch.relu(exp)
        assert float((c0.double() - exp).abs().max() / exp.abs().max()) < (6e-6 if ns == 3 else 6e-5)
