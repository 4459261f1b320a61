"""The template instance and split-K factor each wgmma GEMM launcher picks for a shape, restated in plain Python.

The C entry points choose a kernel instance (operand planes x tile width x pipeline depth x operand layout) and a
split-K factor from the shape alone.  The GPU tests parametrise over shape lists; tests/test_gemm_instances_cpu.py
maps those lists through the rules below and checks that every instance and both sides of every split-K decision are
run.  Each rule names the function of csrc/ and the condition it restates: a change there has to be mirrored here, and
the CPU test then says which shapes the GPU tests are missing.
"""
from __future__ import annotations

SMS = 132       # H100 SXM streaming multiprocessors
BM = 128        # output rows per tile (all three kernels)


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def _pad64(k: int) -> int:
    return _cdiv(k, 64) * 64


# ---------------------------------------------------------------- gemm_sm90.cu
# launch_gemm's split-K rule (gemm_sm90.cu, `if (!relu && !out_half && tiles < sms && nkb_total >= 32)`)
def _nt_ksplit(batch: int, m: int, n: int, bn: int, kpad: int, act: int, out_half: bool, sms: int) -> int:
    tiles = _cdiv(m, BM) * _cdiv(n, bn) * batch
    nkb = kpad // 64
    ksplit = 1
    if not act and not out_half and tiles < sms and nkb >= 32:
        ksplit = _cdiv(2 * sms, tiles)
        ksplit = max(1, min(ksplit, nkb // 8))
        per = _cdiv(nkb, ksplit)
        ksplit = _cdiv(nkb, per)
    return ksplit


# gemm_nt_kernel<NSPLIT, BN, STAGES, FP16, MN> instances of the fp32-plane paths (gemm_sm90.cu: the CODA_GEMM cases of
# coda_gemm_nt_res for nsplit 1-3, the CODA_GEMM_TN cases of coda_gemm_tn)
_PLANE_STAGES = {(1, 64): 6, (1, 128): 6, (2, 64): 4, (2, 128): 3, (3, 64): 2, (3, 128): 2}
# fp16 instances (gemm_sm90.cu: the `if (is_fp16)` CODA_GEMM cases of coda_gemm_nt_res)
_FP16_STAGES = {64: 6, 256: 4, 192: 5, 128: 6}

NT_INSTANCES = {(ns, bn, st, False, False) for (ns, bn), st in _PLANE_STAGES.items()} | \
               {(1, bn, st, True, False) for bn, st in _FP16_STAGES.items()}
TN_INSTANCES = {(ns, bn, st, False, True) for (ns, bn), st in _PLANE_STAGES.items()}


def gemm_nt(nsplit: int, fp16: bool, batch: int, m: int, n: int, k: int, act: int = 0, out_half: bool = False,
            sms: int = SMS):
    """coda_gemm_nt_res -> ((NSPLIT, BN, STAGES, FP16, MN), ksplit)"""
    # tile width (gemm_sm90.cu: `bn` in coda_gemm_nt_res, without the ping-pong case)
    bn = (64 if n <= 64 else 256 if (fp16 and n % 256 == 0 and n >= 1536)
          else 192 if (fp16 and n % 192 == 0 and n >= 384) else 128)
    stages = _FP16_STAGES[bn] if fp16 else _PLANE_STAGES[(nsplit, bn)]
    return (nsplit, bn, stages, fp16, False), _nt_ksplit(batch, m, n, bn, _pad64(k), act, out_half, sms)


def gemm_tn(nsplit: int, mc: int, m: int, n: int, sms: int = SMS):
    """coda_gemm_tn -> ((NSPLIT, BN, STAGES, FP16, MN), ksplit); mc = contraction rows"""
    bn = 64 if n <= 64 else 128                                   # gemm_sm90.cu: `bn` in coda_gemm_tn
    # batch 1, no bias / activation, kpad = mc rounded up to 64 (gemm_sm90.cu: `kpad` and CODA_GEMM_TN in coda_gemm_tn)
    return (nsplit, bn, _PLANE_STAGES[(nsplit, bn)], False, True), _nt_ksplit(1, m, n, bn, _pad64(mc), 0, False, sms)


# ---------------------------------------------------------------- gemm_a32_sm90.cu
A32_PLAIN, A32_AFFINE_RELU, A32_BN_BWD, A32_BN_BWD_POOLED, A32_BN_BWD_POOLED_PRE = 0, 1, 2, 3, 4

# gemm_a32_kernel<NSPLIT, BN, RAW_KB, B_STAGES, B_MN> instances (gemm_a32_sm90.cu: the CODA_A32 cases of coda_gemm_a32),
# each with B K- or MN-major
_A32_BASE = [(2, 64, 128, 4), (2, 128, 128, 2), (3, 64, 128, 3), (3, 128, 64, 3), (3, 128, 96, 2)]
A32_INSTANCES = {base + (mn,) for base in _A32_BASE for mn in (False, True)}


def gemm_a32(nsplit: int, m: int, n: int, k: int, b_mn: bool, mode: int = A32_PLAIN, stats: bool = False,
             sms: int = SMS):
    """coda_gemm_a32 -> ((NSPLIT, BN, RAW_KB, B_STAGES, B_MN), b_resident)"""
    # 64-wide tiles when 128-wide ones would leave half the SMs idle (gemm_a32_sm90.cu: `bn` in coda_gemm_a32)
    tiles128 = _cdiv(m, BM) * _cdiv(n, 128)
    bn = 64 if (n <= 64 or tiles128 <= sms // 2) else 128
    # deep B ring for long contractions (gemm_a32_sm90.cu: `deep_b` in coda_gemm_a32)
    deep_b = not stats and k > 128 and mode != A32_BN_BWD
    if nsplit == 2:
        inst = (2, 64, 128, 4) if bn == 64 else (2, 128, 128, 2)
    elif bn == 64:
        inst = (3, 64, 128, 3)
    else:
        inst = (3, 128, 64, 3) if deep_b else (3, 128, 96, 2)
    # B-resident persistent grid (gemm_a32_sm90.cu: `Q.b_resident` in launch_a32)
    tiles_m, tiles_n, nkb = _cdiv(m, BM), _cdiv(n, bn), _cdiv(k, 64)
    b_resident = nkb <= inst[3] and tiles_n <= sms and tiles_m >= 4 * (sms // tiles_n)
    return inst + (b_mn,), b_resident


# ---------------------------------------------------------------- gemm_tn32_sm90.cu
TN32_INSTANCES = {64, 128}      # gemm_tn32_kernel<BN> (gemm_tn32_sm90.cu: `n <= 64` in coda_gemm_tn32)


def gemm_tn32(rows: int, m: int, n: int, sms: int = SMS):
    """coda_gemm_tn32 -> (BN, ksplit, empty_splits): empty_splits = trailing splits with no 32-row slab"""
    bn = 64 if n <= 64 else 128
    # split-K over the rows, at least four slabs per split (gemm_tn32_sm90.cu: `ksplit` in launch_tn32)
    tiles = _cdiv(m, BM) * _cdiv(n, bn)
    nkb = _cdiv(rows, 32)
    ksplit = max(1, sms // tiles)
    if ksplit > nkb // 4:
        ksplit = max(1, nkb // 4)
    # splits ks with ks * per >= nkb read nothing (gemm_tn32_kernel: `nkb` is 0, the accumulator is zeroed)
    per = _cdiv(nkb, ksplit)
    empty = sum(1 for ks in range(ksplit) if ks * per >= nkb)
    return bn, ksplit, empty
