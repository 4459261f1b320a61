"""The fp16 ping-pong GEMM (gemm_f16_pp_kernel, csrc/gemm_sm90.cu): the CLIP tower's fp16-output GEMMs with at least
two 128-wide tiles per SM.  Its two consumer warpgroups own alternate tiles and issue their main loops in turn.  Every
case runs three times on the same inputs, once right after a launch of another shape, and must give the same bits each
time, match fp64 within the fp16 output rounding, and match bit for bit the fp32-output kernel's C rounded to fp16
(the same k-order in fp32, then the same epilogue)."""
import pytest
import torch

SMS = 132
BM, PP_BN = 128, 128
PP_NONE, PP_BIAS, PP_BIAS_GELU, PP_BIAS_RES = 0, 1, 2, 3
PP_INSTANCES = {(PP_BN, 6, e) for e in (PP_NONE, PP_BIAS, PP_BIAS_GELU, PP_BIAS_RES)}


def pp_instance(m: int, n: int, bias: bool, act: int, res: bool, ldc_pad: int = 0, sms: int = SMS):
    """coda_gemm_nt_res's rule for an fp16-output, batch-1 call with aligned operands -> (BN, STAGES, EPI) of the
    ping-pong kernel, or None where gemm_nt_kernel (tests/gemm_instances.py) runs it."""
    if bias:
        epi = (PP_BIAS_RES if res else PP_BIAS) if act == 0 else (PP_BIAS_GELU if act == 2 and not res else None)
    else:
        epi = PP_NONE if act == 0 and not res else None
    tiles = -(-m // BM) * (n // PP_BN)
    if epi is None or n % PP_BN or tiles < 2 * sms or (n + ldc_pad) % 8:
        return None
    return PP_BN, 6, epi


# (m, n, k, bias, act, residual, ldc_pad)
TOWER = [
    (12800, 2304, 768, True, 0, False, 0),      # qkv
    (12800, 768, 768, True, 0, True, 0),        # out_proj + residual
    (12800, 3072, 768, True, 2, False, 0),      # c_fc + QuickGELU
    (12800, 768, 3072, True, 0, True, 0),       # c_proj + residual
    (12544, 768, 3072, False, 0, False, 0),     # patch embedding
    (12800, 512, 768, False, 0, False, 0),      # _project
]
EDGES = [
    (8448, 512, 128, True, 0, False, 0),        # 264 tiles: one per warpgroup on 132 SMs
    (8300, 640, 192, True, 2, False, 0),        # ragged m, 325 tiles: 3 or 2 per CTA
    (8300, 640, 64, True, 0, True, 8),          # one k-block per tile, ldc > n
    (4000, 1024, 256, False, 0, False, 0),      # 256 tiles: below two per SM, gemm_nt_kernel
    (12800, 768, 768, True, 1, False, 0),       # ReLU: gemm_nt_kernel
    (12800, 768, 256, True, 0, False, 3),       # ldc not a multiple of 8: gemm_nt_kernel
]
CASES = TOWER + EDGES


def test_cases_reach_every_instance_and_both_sides_of_the_rule():
    picks = [pp_instance(m, n, bias, act, res, pad) for m, n, k, bias, act, res, pad in CASES]
    assert {p for p in picks if p} == PP_INSTANCES
    assert any(p is None for p in picks)
    assert all(pp_instance(m, n, bias, act, res) for m, n, k, bias, act, res, _ in TOWER)
    # tiles per CTA of the persistent grid (SMS CTAs): one tile per warpgroup, and odd and even counts above that
    per_cta = set()
    for m, n, k, bias, act, res, pad in CASES:
        if pp_instance(m, n, bias, act, res, pad):
            tiles = -(-m // BM) * (n // PP_BN)
            per_cta |= {tiles // SMS, -(-tiles // SMS)}
    assert 2 in per_cta and any(c % 2 for c in per_cta) and any(c % 2 == 0 and c > 2 for c in per_cta)


def _inputs(m, n, k, bias, res, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(1, 1, m, k, device="cuda", generator=g) * 0.5).half()
    b = (torch.randn(1, 1, n, k, device="cuda", generator=g) * k ** -0.5).half()
    bv = torch.randn(n, device="cuda", generator=g) if bias else None
    r = torch.randn(m, n, device="cuda", generator=g).half() if res else None
    return a, b, bv, r


def _run(a, b, m, n, bv, act, r, pad):
    from coda_neurips2023_b200 import ops

    full = torch.zeros(1, m, n + pad, device="cuda", dtype=torch.float16)
    return ops.gemm_nt(a, b, m, n, bias=bv, act=act, out=full[..., :n], residual=r)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k,bias,act,res,pad", CASES)
def test_same_bits_every_call_and_vs_fp64(built_lib, m, n, k, bias, act, res, pad):
    from coda_neurips2023_b200 import ops

    a, b, bv, r = _inputs(m, n, k, bias, res, seed=m + n + k)
    c0 = _run(a, b, m, n, bv, act, r, pad)
    c1 = _run(a, b, m, n, bv, act, r, pad)
    om, on, ok, obias, oact, ores, opad = TOWER[0] if (m, n) != (12800, 2304) else TOWER[1]
    _run(*_inputs(om, on, ok, obias, ores, seed=1)[:2], om, on, None, 0, None, 0)   # another grid in between
    c2 = _run(a, b, m, n, bv, act, r, pad)
    assert torch.equal(c0, c1) and torch.equal(c0, c2)

    # the fp32-output kernel sums in the same order: its C + residual, rounded once, has the same bits
    c32 = ops.gemm_nt(a, b, m, n, bias=bv, act=act)[0]
    assert torch.equal(c0, (c32 + r.float() if res else c32).half())

    ref = a[0, 0].double() @ b[0, 0].double().t()
    if bias:
        ref = ref + bv.double()
    if act == 1:
        ref = ref.relu()
    if act == 2:
        ref = ref * torch.sigmoid(1.702 * ref)
    if res:
        ref = ref + r.double()
    assert ((c0.double() - ref).abs().max() / ref.abs().max()).item() < 2e-3     # fp16 output rounding
