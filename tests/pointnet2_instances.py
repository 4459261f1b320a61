"""The kernel instance, cluster width, tile count and channel split each PointNet++ launcher picks, restated in Python.

coda_furthest_point_sampling picks a register-resident fps_cluster_kernel<PPT> instance and a thread-block-cluster
width from the scene size (or the generic one-CTA kernel when the scene does not fit); ball_query_impl streams the
scene through shared memory in BQ_TILE-point tiles and refuses an nsample whose hit lists do not fit; the group and
interpolate launchers split channels over blockIdx.y with pick_c_per_block.  The GPU tests parametrise over case lists;
tests/test_pointnet2_instances_cpu.py maps those lists through the rules below and checks that every instance and cell
and both sides of every switch are run.  Each rule names the function of csrc/pointnet2_kernels.cu it restates: a change
there has to be mirrored here, and the CPU test then says which cases the GPU tests are missing.
"""
from __future__ import annotations

import math
import re
from pathlib import Path

KERNELS = Path(__file__).resolve().parent.parent / "coda_neurips2023_b200" / "csrc" / "pointnet2_kernels.cu"

SMS = 132               # H100 SXM streaming multiprocessors (pick_c_per_block aims at 8 CTAs per SM)
FPS_T = 512             # threads per FPS CTA
FPS_MAX_PPT = 16        # most points a thread of fps_cluster_kernel keeps in registers
FPS_WIDTHS = (1, 2, 4, 8)
BQ_WARPS = 8            # ball-query centres per CTA (one warp each)
BQ_TILE = 2048          # scene points per shared-memory tile
BQ_SMEM_MAX = 200 * 1024


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def fps_instances() -> tuple[int, ...]:
    """The PPT of every fps_cluster_kernel instance coda_furthest_point_sampling dispatches to, read from its
    `CODA_FPS_CASE(...)` lines, in dispatch order."""
    return tuple(int(p) for p in re.findall(r"^\s*CODA_FPS_CASE\((\d+)\)", KERNELS.read_text(), flags=re.M))


def fps_block_size_log2(n: int) -> int:
    """ref_block_size_log2: the reference launcher's block size, which defines the tie rule (same double expression)."""
    pow_2 = int(math.log(float(n)) / math.log(2.0))
    if (1 << pow_2) > 512:
        pow_2 = 9
    return pow_2


def fps_path(n: int, forced: int = 0, instances: tuple[int, ...] | None = None):
    """coda_furthest_point_sampling -> (PPT instance, cluster width) or "generic".

    forced is the width set by coda_fps_set_cluster (0: automatic, one CTA up to 4096 positions, else 8)."""
    bs_log2 = fps_block_size_log2(n)
    P = _cdiv(n, 1 << bs_log2) << bs_log2
    cl = forced or (1 if P <= 4096 else 8)
    cl_log2 = (cl - 1).bit_length()
    ppt = _cdiv(P, FPS_T << cl_log2)
    if ppt > FPS_MAX_PPT and cl_log2 < 3:      # a forced width too narrow for the scene is widened to 8
        cl_log2 = 3
        ppt = _cdiv(P, FPS_T << 3)
    if ppt > FPS_MAX_PPT:
        return "generic"
    for inst in instances or fps_instances():
        if ppt <= inst:
            return inst, 1 << cl_log2
    raise AssertionError(f"no FPS instance holds {ppt} points per thread")


def fps_cta_of(pos, width: int):
    """Rank, within its cluster, of the CTA holding position `pos` (fps_cluster_kernel deals positions round-robin
    to the width * FPS_T threads of the cluster)."""
    return (pos % (width * FPS_T)) // FPS_T


def bq_tiles(n: int) -> int:
    """Shared-memory tiles ball_query_kernel streams for a scene of n points."""
    return _cdiv(n, BQ_TILE)


def bq_max_nsample() -> int:
    """Largest nsample ball_query_impl accepts: one tile plus BQ_WARPS hit lists in BQ_SMEM_MAX bytes."""
    return (BQ_SMEM_MAX - BQ_TILE * 3 * 4) // (BQ_WARPS * 4)


def c_per_block(c: int, work_items_per_channel: int, b: int) -> int:
    """pick_c_per_block: channels per blockIdx.y slice of the group / interpolate kernels."""
    ctas_per_slice = _cdiv(work_items_per_channel, 256) * b
    slices = max(1, _cdiv(SMS * 8, ctas_per_slice))
    slices = min(slices, c)
    return _cdiv(c, slices)


def ragged_last_slice(c: int, work_items_per_channel: int, b: int) -> bool:
    """The last channel slice is shorter than the others."""
    return c % c_per_block(c, work_items_per_channel, b) != 0
