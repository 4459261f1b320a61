"""What the CLIP crop kernel and the novel-box candidate kernel run for a shape, restated in plain Python.

coda_crop_resize_normalize_ex (csrc/image_kernels.cu) picks a tile height and a shared-memory carve-up from the image
size and the resolution, sizes every filter from the box, and takes one of three branches for every resampled source
row; coda_novel_candidates (csrc/discovery_kernels.cu) sizes its shared memory from q.  tests/test_crop_discovery_paths_cpu.py
uses these rules to prove that the crop kernel's tap cap and its direct-form fallback never come into play, pins the
ScanNet plan, and maps the case lists of the GPU tests through them to check that every path and edge is run.  Each
rule names the lines it restates: a change there has to be mirrored here, and the CPU test then says which cases the
GPU tests are missing.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

F32 = np.float32

# ------------------------------------------------------------------ crop / pad / resize (image_kernels.cu)
MAX_TAPS = 40                  # image_kernels.cu:14
CR_SMEM_LIMIT = 220 * 1024     # image_kernels.cu:35
AUTO_TILE_ROWS = 16            # the automatic plan starts here (image_kernels.cu:214)
MAX_TILE_ROWS = 64             # image_kernels.cu:251
MAX_CROPS = 65535              # one crop per grid row (image_kernels.cu:232, :254)


@dataclass(frozen=True)
class CropPlan:
    tr: int        # output rows per CTA
    rmax: int      # source rows the shared buffer holds
    taps: int      # per-axis tap cap (xt == yt)
    smem: int      # dynamic shared memory, bytes


def crop_plan(h: int, w: int, res: int, tile_rows: int = 0):
    """the launch plan for the largest box an (h, w) image holds, or None for CODA_ETOOLARGE (image_kernels.cu:209-223,
    refused at :259): taps per axis from the largest scale, then the tile height halves from `tile_rows` (16 when 0)
    until the carve-up fits CR_SMEM_LIMIT.  Host arithmetic in fp32 like the source."""
    ms = max(F32(max(h, w)) / F32(res), F32(1.0))
    taps = 2 * int(np.ceil(F32(2.0) * ms)) + 1
    if taps > MAX_TAPS:
        return None
    tr = tile_rows if tile_rows > 0 else AUTO_TILE_ROWS
    while tr >= 1:
        rmax = int(np.ceil(F32(tr) * ms)) + 2 * int(np.ceil(F32(2.0) * ms)) + 3
        smem = (rmax * res * 3 + res * taps + tr * taps) * 4 + (2 * res + 2 * tr) * 4
        if smem <= CR_SMEM_LIMIT:
            return CropPlan(tr, rmax, taps, smem)
        tr >>= 1
    return None


def crop_status(h: int, w: int, res: int, ncrops: int, tile_rows: int = 0) -> str:
    """'ok', 'empty' (launches nothing), 'einval' or 'etoolarge' for the arguments the GPU tests vary
    (image_kernels.cu:250-259)"""
    if ncrops < 0 or res <= 0 or tile_rows < 0 or tile_rows > MAX_TILE_ROWS:
        return "einval"
    if ncrops == 0:
        return "empty"
    if ncrops > MAX_CROPS:
        return "einval"
    return "ok" if crop_plan(h, w, res, tile_rows) is not None else "etoolarge"


def _fma32(a, b, c):
    """fp32 fma: the product of two fp32 values and its sum with an fp32 value of like magnitude are exact in fp64,
    so one rounding to fp32 is the fused result"""
    return (np.float64(a) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def aa_span(edge: int, res: int, fused: bool = False):
    """-> (lo, n) int64 arrays over the `res` output indices: the first source index and the tap count of each filter,
    before the cap (image_kernels.cu:55-59).  The compiled kernel rounds `center` before adding the support; `fused`
    evaluates center -/+ support as one fma instead, which a compiler may make of the source.  The two readings
    differ for a few filters, so the CPU proofs are run under both."""
    scale = F32(edge) / F32(res)
    support = F32(2.0) * scale if scale >= 1 else F32(2.0)
    x = np.arange(res, dtype=F32) + F32(0.5)
    if fused:
        lo_arg = _fma32(scale, x, -support) + F32(0.5)
        hi_arg = _fma32(scale, x, support) + F32(0.5)
    else:
        center = scale * x
        lo_arg = center - support + F32(0.5)
        hi_arg = center + support + F32(0.5)
    lo = np.maximum(lo_arg.astype(np.int64), 0)          # (int) truncates toward zero
    n = np.minimum(hi_arg.astype(np.int64), edge) - lo
    return lo, n


def crop_geometry(box):
    """-> (wc, hc, edge, x_begin, y_begin) of a box [xmin, ymin, xmax, ymax] (image_kernels.cu:105-108)"""
    xmin, ymin, xmax, ymax = (int(v) for v in box)
    wc, hc = xmax - xmin, ymax - ymin
    edge = max(wc, hc)
    return wc, hc, edge, (edge - wc) // 2, (edge - hc) // 2


def tile_nsrc(lo, n, tr: int, taps: int):
    """source rows each tile of `tr` output rows touches (image_kernels.cu:122-123), with the taps capped like
    aa_weights_to (:60)"""
    res = len(lo)
    end = lo + np.minimum(n, taps)
    starts = np.arange(0, res, tr)
    lasts = np.minimum(starts + tr, res) - 1
    return end[lasts] - lo[starts]


def hrow_branches(box, res: int) -> set:
    """which branches of hrow (image_kernels.cu:132-164) a crop's horizontal pass takes, over every source row its
    tiles touch and every output column: 'inside' (every tap in the pasted crop, :140), 'white' (a row of the white
    canvas, :149) and 'mixed' (taps on both, :153).  The x and y filters of a crop are the same (:113, :118)."""
    wc, hc, edge, xb, yb = crop_geometry(box)
    lo, n = aa_span(edge, res)
    cy = np.arange(lo[0], lo[-1] + n[-1]) - yb        # the tiles' source rows cover this range without a gap
    yin = (cy >= 0) & (cy < hc)
    c0 = lo - xb
    xin = (c0 >= 0) & (c0 + n <= wc)
    out = set()
    if yin.any() and xin.any():
        out.add("inside")
    if (~yin).any():
        out.add("white")
    if yin.any() and (~xin).any():
        out.add("mixed")
    return out


# ------------------------------------------------------------------ novel-box candidates (discovery_kernels.cu)
NC_MAXQ = 1024                 # discovery_kernels.cu:19
NC_THREADS = 256               # discovery_kernels.cu:21, :151
NC_SMEM_CAP = 200 * 1024       # discovery_kernels.cu:148


def novel_candidates_layout(q: int) -> dict:
    """byte offset of each shared-memory array: box (float4), score, order, suppression rows, keep words and flags
    (discovery_kernels.cu:26-34)"""
    words = (q + 31) // 32
    off, out = 0, {}
    for name, size in (("box", 16 * q), ("score", 4 * q), ("order", 4 * q), ("sup", 4 * q * words),
                       ("keep", 4 * words), ("ok", q)):
        out[name] = off
        off += size
    return out


def novel_candidates_smem(q: int) -> int:
    """the dynamic shared memory the launcher asks for: the arrays above and 16 bytes (discovery_kernels.cu:147)"""
    words = (q + 31) // 32
    return q * (4 + 16 + 4) + q * words * 4 + words * 4 + q + 16


def novel_candidates_status(b: int, q: int, g: int, cap: int) -> str:
    """'ok', 'empty' (b == 0), 'einval' or 'etoolarge' (discovery_kernels.cu:142-148)"""
    if b < 0 or q < 1 or q > NC_MAXQ or g < 0 or cap < 1:
        return "einval"
    if b == 0:
        return "empty"
    return "ok" if novel_candidates_smem(q) <= NC_SMEM_CAP else "etoolarge"
