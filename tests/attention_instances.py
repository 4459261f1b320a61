"""The template instance, ring depth and tile walk of each wgmma attention kernel for a shape, restated in plain Python.

The C entry points of csrc/attention_sm90.cu (forward) and csrc/attention_bwd_sm90.cu (dQ and dK/dV kernels) pick a
kernel instance from the head dim, the operand planes and the query length.  Each instance streams 64-row tiles
through a ring of NST shared-memory stages whose mbarrier phase flips every time the ring wraps.  The GPU tests
parametrise over shape lists; tests/test_attention_instances_cpu.py maps those lists through the rules below and
checks that every instance, tail and ring wrap is run.  Each rule names the definition and condition it restates: a
change there has to be mirrored here, and the CPU test then says which shapes the GPU tests are missing.
"""
from __future__ import annotations

KT = 64                 # keys (forward, dQ) or queries (dK/dV) per streamed tile (attention_common.cuh: attn::KT)
SMEM = 220 * 1024       # shared memory the ring depth is fitted into (NST_FIT of AttnCfg and BwdCfg)
BOX = 64 * 128          # one [64 rows x 64] 16-bit TMA box


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


# ---------------------------------------------------------------- attention_sm90.cu
def fwd_nst(hd: int, nsplit: int, nwg: int) -> int:
    """AttnCfg<HD, NSPLIT, NWG>::NST (attention_sm90.cu)"""
    kb = hd // 64
    q_bytes = nsplit * nwg * kb * BOX
    stage = 2 * nsplit * kb * BOX
    return max(1, min(4, (SMEM - q_bytes) // stage))


def fwd_instance(lq: int, hd: int, nsplit: int, f16: bool = False):
    """launch_attn -> attn_fwd_kernel<HD, NSPLIT, NWG, F16>: one warpgroup for Lq <= 64 or head dim 128
    (launch_attn: `one = Lq <= 64 || HD == 128`).  coda_attention_fwd_half runs <64, 1, *, true> on l <= 64."""
    assert not f16 or (hd == 64 and nsplit == 1 and lq <= KT)
    nwg = 1 if (lq <= 64 or hd == 128) else 2
    return hd, nsplit, nwg, f16


FWD_INSTANCES = {(hd, ns, nwg, False) for hd in (64, 128) for ns in (1, 2, 3) for nwg in (1, 2)
                 if not (hd == 128 and nwg == 2)} | {(64, 1, 1, True)}


def half_out_accepted(lk: int, hd: int, nsplit: int, masked: bool) -> bool:
    """coda_attention_fwd_packed_masked accepts out_half only for one key tile at hd 64, <= 2 planes, no mask
    (its `if (out_half && ...)` check); any other combination returns CODA_EINVAL."""
    return hd == 64 and lk <= KT and nsplit <= 2 and not masked


def half_out_requested(lk: int, hd: int, nsplit: int) -> bool:
    """attention_launch.forward passes half_out through only where the kernel has it (attention_launch.py:102): the
    mask is not part of the Python rule, so a masked call asking for half output reaches the C check."""
    return lk <= KT and hd == 64 and nsplit <= 2


# ---------------------------------------------------------------- attention_bwd_sm90.cu
def bwd_nwg(hd: int) -> int:
    """launch_bwd: two MMA warpgroups at head dim 64, one at 128, for both kernels (`NWG = HD == 64 ? 2 : 1`)"""
    return 2 if hd == 64 else 1


def bwd_nst(hd: int) -> int:
    """BwdCfg<HD, NWG>::NST (attention_bwd_sm90.cu)"""
    kb, nwg = hd // 64, bwd_nwg(hd)
    res = 2 * 2 * nwg * kb * BOX            # K and V (or Q and dO) rows, two planes each
    stage = 2 * 2 * kb * BOX
    return min(4, (SMEM - res) // stage)


BWD_INSTANCES = {(64, 2), (128, 1)}


def bwd_instance(hd: int):
    return hd, bwd_nwg(hd)


def lqp(lq: int) -> int:
    """rows of the padded (lse log2 e, D) array the dK/dV kernel bulk-loads one 64-query tile at a time
    (attention_bwd_sm90.cu: `lqp` of the qv array, bulk-loaded by attn_bwd_dkv_kernel)"""
    return _cdiv(lq, 64) * 64


# ---------------------------------------------------------------- the walk of one kernel over a shape
def tiles(n: int) -> int:
    """streamed 64-row tiles (`ntiles` of attn_fwd_kernel, attn_bwd_dq_kernel and attn_bwd_dkv_kernel)"""
    return _cdiv(n, KT)


def tail(n: int) -> bool:
    """the last streamed tile is partial (padded rows are zero-filled by TMA and masked by `col >= kvalid`)"""
    return n % KT != 0


def wraps(n: int, nst: int) -> int:
    """times a ring of nst stages wraps over n rows: stage j % nst waits on phase (j / nst) & 1, so one wrap flips the
    phase and two bring it back"""
    return (tiles(n) - 1) // nst


def row_tail_warpgroup(n: int, nwg: int):
    """warpgroup of a (64 * nwg)-row CTA that holds the last valid row of the last CTA, or None when the CTA is full;
    with nwg = 2, a tail in warpgroup 0 leaves warpgroup 1 without a single valid row"""
    r = n % (64 * nwg)
    return None if r == 0 else (r - 1) // 64


def fwd_walk(lq: int, lk: int, hd: int, nsplit: int) -> dict:
    inst = fwd_instance(lq, hd, nsplit)
    nst = fwd_nst(hd, nsplit, inst[2])
    return dict(instance=inst, nst=nst, key_tiles=tiles(lk), key_tail=tail(lk), wraps=wraps(lk, nst),
                q_tail_wg=row_tail_warpgroup(lq, inst[2]))


def bwd_walk(lq: int, lk: int, hd: int) -> dict:
    """dQ: CTA of 64 NWG queries over the key tiles; dK/dV: CTA of 64 NWG keys over the query tiles"""
    nwg, nst = bwd_nwg(hd), bwd_nst(hd)
    return dict(instance=(hd, nwg), nst=nst, dq_tiles=tiles(lk), dq_wraps=wraps(lk, nst), dkv_tiles=tiles(lq),
                dkv_wraps=wraps(lq, nst), q_tail=tail(lq), k_tail=tail(lk), lqp=lqp(lq),
                q_tail_wg=row_tail_warpgroup(lq, nwg), k_tail_wg=row_tail_warpgroup(lk, nwg))
