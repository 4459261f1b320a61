"""What the step's glue kernels run for a shape, and which elements their dropout keeps, restated in plain Python.

The LayerNorm family (csrc/detr_kernels.cu), the kernels of csrc/step_kernels.cu and the Hungarian matcher pick an
instance, a grid, a scalar head / tail or a shared-memory layout from the shape alone.  tests/test_step_glue_paths_cpu.py
maps the case lists of the GPU tests through the rules below and checks that every instance and every edge is run.
Each rule names the lines it restates: a change there has to be mirrored here, and the CPU test then says which cases
the GPU tests are missing.

`drop_keep` is a numpy twin of the counter-based dropout mask (`Drop`, step_kernels.cu:17-42): the GPU tests compare
the kernels' masks with it element by element.
"""
from __future__ import annotations

import numpy as np

THREADS = 256                  # step_kernels.cu:14
NUM_SMS = 132                  # step_kernels.cu:15
STREAM_CAP = NUM_SMS * 8       # stream_grid's cap (step_kernels.cu:46)
BN_MAX_BLOCKS = NUM_SMS * 4    # grid_for's cap (step_kernels.cu:92)
NORM_BLOCKS = NUM_SMS * 4      # step_kernels.cu:203
LN_WARPS = 8                   # rows per forward block (detr_kernels.cu:30, :53)
LN_BWD_ROWS = 64               # LN_BWD_ROWS_PER_BLOCK (detr_kernels.cu:141)
HUNG_SMEM_CAP = 200 * 1024     # detr_kernels.cu:683-684

# every width channels_ok accepts: c % 4 == 0 and c / 4 divides 256 (step_kernels.cu:91)
BN_WIDTHS = tuple(4 << i for i in range(9))   # 4, 8, ..., 1024


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


# ------------------------------------------------------------------ LayerNorm (detr_kernels.cu)
def ln_instance(c: int):
    """the NV of layer_norm_{fwd,fwd_half,bwd}_kernel<NV>, or None when the entry points refuse c
    (detr_kernels.cu:555, :565-568, :581, :589-592, :606, :620-623)"""
    if c <= 0 or c % 128 or c > 1024:
        return None
    return c // 128


def ln_fwd_grid(rows: int) -> int:
    """one warp per row, 8 rows per block (detr_kernels.cu:53, :560, :584)"""
    return _cdiv(rows, LN_WARPS)


def ln_bwd_blocks(rows: int) -> int:
    """64 rows per block (detr_kernels.cu:164-167, :616); rows == 0 launches nothing and zero-fills dgamma / dbeta
    (detr_kernels.cu:608-612)"""
    return _cdiv(rows, LN_BWD_ROWS)


def ln_bwd_last_block_rows(rows: int) -> int:
    """rows the last backward block walks before its `row >= rows` break (detr_kernels.cu:165-167)"""
    return rows - LN_BWD_ROWS * (ln_bwd_blocks(rows) - 1) if rows > 0 else 0


# ------------------------------------------------------------------ BatchNorm on rows (step_kernels.cu)
def bn_channels_ok(c: int) -> bool:
    """step_kernels.cu:91"""
    return 4 <= c <= 1024 and c % 4 == 0 and THREADS % (c // 4) == 0


def bn_slots(c: int) -> int:
    """rows in flight per block iteration: a thread owns 4 channels (step_kernels.cu:112, :130, :184)"""
    return THREADS // (c // 4)


def bn_grid(rows: int, c: int) -> int:
    """grid_for (step_kernels.cu:93-97)"""
    return min(max(_cdiv(rows, bn_slots(c)), 1), BN_MAX_BLOCKS)


def bn_strided(rows: int, c: int) -> bool:
    """the row loop of the forward, reduce and backward kernels takes a second grid-stride step"""
    return rows > bn_grid(rows, c) * bn_slots(c)


# ------------------------------------------------------------------ streaming kernels: dropout, n-ary sum
def stream_grid(work_items: int) -> int:
    """step_kernels.cu:44-48; dropout_add and sum_n pass n / 4 + 1 (step_kernels.cu:390, :470)"""
    return min(max(_cdiv(work_items, THREADS), 1), STREAM_CAP)


def stream_strided(n: int) -> bool:
    """the float4 loop of dropout_add_kernel / sum_n_kernel takes a second grid-stride step (step_kernels.cu:55, :302)"""
    return n // 4 > stream_grid(n // 4 + 1) * THREADS


def scalar_tail(n: int) -> int:
    """elements block 0 handles one by one after the float4 loop (step_kernels.cu:64-67, :214-217, :310-315)"""
    return n & 3


# ------------------------------------------------------------------ clip + AdamW (step_kernels.cu)
def norm_grid(n: int) -> int:
    """sumsq_partial_kernel's grid (step_kernels.cu:441-442)"""
    return min(max(_cdiv(n // 4, THREADS), 1), NORM_BLOCKS)


def norm_strided(n: int) -> bool:
    """sumsq_partial_kernel's float4 loop takes a second grid-stride step (step_kernels.cu:210)"""
    return n // 4 > norm_grid(n) * THREADS


def adamw_split(offset: int, length: int):
    """-> (head, body4, tail): scalar elements before the 16-byte aligned body, float4s of the body and scalar
    elements after it, for one chunk (step_kernels.cu:264, :273, :283-284)"""
    head = min((4 - (offset & 3)) & 3, length)
    body4 = (length - head) >> 2
    return head, body4, length - head - 4 * body4


# ------------------------------------------------------------------ Hungarian (detr_kernels.cu)
def hungarian_smem_bytes(nr_max: int, nc_max: int, stage_cost: bool) -> int:
    """detr_kernels.cu:394-401"""
    s = 8 * (nr_max + 2 * nc_max) + 4 * (3 * nc_max + nr_max) + (nr_max + nc_max + 15) // 16 * 16
    if stage_cost:
        s += 4 * nr_max * nc_max
    return s + 64


def hungarian_staged(nprop: int, ngt: int) -> bool:
    """the cost matrix is copied to shared memory when it fits in 200 KiB beside the solver's arrays, else read from
    global memory (detr_kernels.cu:680-684); None when even the unstaged layout does not fit (CODA_ETOOLARGE)"""
    lo, hi = min(nprop, ngt), max(nprop, ngt)
    if hungarian_smem_bytes(lo, hi, True) <= HUNG_SMEM_CAP:
        return True
    return False if hungarian_smem_bytes(lo, hi, False) <= HUNG_SMEM_CAP else None


def hungarian_scene(nprop: int, ngt: int, nactual: int):
    """-> (na, transposed) of one scene: nactual clamped to ngt (detr_kernels.cu:414-416); the problem is solved as
    gt x proposals when there are more proposals than matched columns (detr_kernels.cu:418-420)"""
    na = min(nactual, ngt)
    return na, (na < nprop if na > 0 else None)


# ------------------------------------------------------------------ the dropout mask (step_kernels.cu:17-42)
_M32 = np.uint64(0xFFFFFFFF)


def mix32(x):
    """lowbias32-style avalanche on uint32 values held in uint64 (step_kernels.cu:20-25)"""
    x = np.asarray(x, dtype=np.uint64) & _M32
    x = x ^ (x >> np.uint64(16))
    x = (x * np.uint64(0x7FEB352D)) & _M32
    x = x ^ (x >> np.uint64(15))
    x = (x * np.uint64(0x846CA68B)) & _M32
    return x ^ (x >> np.uint64(16))


def drop_threshold(p: float) -> int:
    """(uint32)fminf(p * 2^32, 4294967040) with p and the product in fp32 (step_kernels.cu:33)"""
    t = np.minimum(np.float32(p) * np.float32(4294967296.0), np.float32(4294967040.0))
    return int(t)


def drop_scale(p: float) -> np.float32:
    """1 / (1 - p) in fp32 (step_kernels.cu:34)"""
    return np.float32(1.0) / (np.float32(1.0) - np.float32(p))


def drop_keep(seed: int, salt: int, p: float, index) -> np.ndarray:
    """bool keep mask of the elements `index` (int array) of a call with device seed `seed` and call-site `salt`
    (step_kernels.cu:30-41); p == 0 keeps everything"""
    index = np.asarray(index, dtype=np.uint64)
    if not p > 0.0:
        return np.ones(index.shape, dtype=bool)
    key = mix32((np.uint64(seed & 0xFFFFFFFF) + np.uint64(salt & 0xFFFFFFFF) * np.uint64(0x9E3779B1)) & _M32)
    lo, hi = index & _M32, index >> np.uint64(32)
    inner = mix32((lo * np.uint64(0x85EBCA77) + hi * np.uint64(0xC2B2AE3D) + np.uint64(0x27D4EB2F)) & _M32)
    return mix32(key ^ inner) >= np.uint64(drop_threshold(p))
