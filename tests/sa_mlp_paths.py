"""Which kernels, instances and backward branch the fused shared-MLP + max-pool node runs for a shape, restated in
plain Python.

`sa_mlp._SharedMLPMax` picks the first-layer kernel, the backward branch of its last layer and the grids of the row
kernels of csrc/sa_mlp_kernels.cu from the shape alone.  tests/test_sa_mlp_paths_cpu.py maps the case lists of
tests/test_sa_mlp_edges_gpu.py through the rules below and checks that every small-K instance, every channel width,
every backward branch and every grid-strided loop is run.  Each rule names the definition it restates: a change there
has to be mirrored here, and the CPU test then says which cases the GPU tests are missing.
"""
from __future__ import annotations

THREADS = 256                 # threads per row-kernel block (sa_mlp_kernels.cu: THREADS)
MAX_BLOCKS = 132 * 4          # grid_for's cap (sa_mlp_kernels.cu: MAX_BLOCKS)
MAXPOOL_BLOCKS = 132 * 8      # coda_bn_relu_maxpool_rows's cap (sa_mlp_kernels.cu: its `grid`)
COLSUM_BLOCKS = 132           # coda_rows_colsum's cap on grid_for (sa_mlp_kernels.cu: `if (grid > 132)`)

# every width _channels_ok accepts: c % 4 == 0 and c / 4 divides 256
WIDTHS = tuple(4 << i for i in range(9))      # 4, 8, ..., 1024


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def channels_ok(c: int) -> bool:
    """sa_mlp.py:33-34, sa_mlp_kernels.cu: channels_ok"""
    return 4 <= c <= 1024 and c % 4 == 0 and 256 % (c // 4) == 0


def applicable(cin: int, widths, group: int, x_grad: bool) -> bool:
    """sa_mlp.applicable (sa_mlp.py:37-56) for fp32 CUDA rows, bias-free convolutions and affine BatchNorm in
    training mode; x_grad: the input requires a gradient with autograd enabled"""
    if not 1 <= group <= 256 or len(widths) == 0:
        return False
    if cin > 8 and cin % 64 != 0:
        return False
    if cin <= 8 and x_grad:
        return False
    # every layer but a small-K first one is a GEMM whose column statistics fit beside its stages up to 256 columns
    return all(channels_ok(c) and (li == len(widths) - 1 or c % 64 == 0) and (c <= 256 or (li == 0 and cin <= 8))
               for li, c in enumerate(widths))


def small_k(cin: int):
    """the linear_small_k_kernel / bn_relu_bwd_small_k_kernel instance of the first layer, or None for the wgmma
    GEMM (sa_mlp.py:149; the CODA_CASE instances of coda_rows_linear_small_k and coda_bn_relu_bwd_small_k)"""
    return cin if cin <= 8 else None


def pooled_pre(group: int, cout: int) -> bool:
    """the last layer's gradient GEMMs place the pooled gradient in their prologue (sa_mlp.py:260)"""
    return group % 32 == 0 and (128 % group == 0 or group % 128 == 0) and cout % 128 == 0


def backward_branches(cin: int, widths, group: int) -> set:
    """branches _SharedMLPMax.backward takes (sa_mlp.py:213-277):
    "single_block_expand"  one small-K block: the pooled gradient is expanded for bn_relu_bwd_small_k (line 238)
    "pooled_pre"           last layer through A32_BN_BWD_POOLED_PRE (line 260)
    "expand"               last layer's pooled gradient expanded once, then A32_BN_BWD (lines 264-269)
    "small_k"              first layer through bn_relu_bwd_small_k under a GEMM layer (line 237)"""
    if small_k(cin) is not None and len(widths) == 1:
        return {"single_block_expand"}
    out = {"pooled_pre" if pooled_pre(group, widths[-1]) else "expand"}
    if small_k(cin) is not None:
        out.add("small_k")
    return out


def slots(c: int) -> int:
    """rows in flight per block iteration: a thread owns 4 channels (sa_mlp_kernels.cu: `nslots` of the row kernels)"""
    return THREADS // (c // 4)


def grid_for(rows: int, c: int) -> int:
    """sa_mlp_kernels.cu: grid_for"""
    return min(max(_cdiv(rows, slots(c)), 1), MAX_BLOCKS)


def maxpool_grid(groups: int) -> int:
    """one block iteration per group (bn_relu_maxpool_kernel, coda_bn_relu_maxpool_rows)"""
    return min(groups, MAXPOOL_BLOCKS)


def strided(rows: int, c: int) -> bool:
    """a grid_for-launched kernel whose grid-stride loop takes a second iteration"""
    return rows > grid_for(rows, c) * slots(c)


def colsum_grid(rows: int, c: int) -> int:
    """sa_mlp_kernels.cu: the grid of colsum_partial_kernel in coda_rows_colsum"""
    return min(grid_for(rows, c), COLSUM_BLOCKS)


def colsum_strided(rows: int, c: int) -> bool:
    """colsum_partial_kernel's grid-stride loop takes a second iteration"""
    return rows > colsum_grid(rows, c) * slots(c)


def node_launches(cin: int, widths, b: int, npoint: int, group: int):
    """-> [(kernel, rows, c, grid-strided)] of the row kernels one forward + backward of the node launches"""
    rows, groups = b * npoint * group, b * npoint
    out = []
    if small_k(cin) is not None:
        c0 = widths[0]
        out += [("linear_small_k", rows, c0, strided(rows, c0)), ("stats", rows, c0, strided(rows, c0)),
                ("bwd_small_k", rows, c0, strided(rows, c0))]
    last = widths[-1]
    out += [("maxpool", groups, last, groups > maxpool_grid(groups)),
            ("reduce_pooled", groups, last, strided(groups, last))]
    out += [("reduce", rows, c, strided(rows, c)) for c in widths[:-1]]
    return out
