"""Launchers of the wgmma attention forward and backward (include/coda_attention.h) and the
torch-side twin of their counter-based dropout mask (used by the tests to build the same mask)."""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from ._lib import check, lib, ptr, stream_of

_SEED_DEV: dict = {}   # device -> uint32 step counter living on the device
_CALL_SALT = 0


def seed_counter(device) -> torch.Tensor:
    key = str(device)
    if key not in _SEED_DEV:
        _SEED_DEV[key] = torch.zeros(1, dtype=torch.int32, device=device)
    return _SEED_DEV[key]


def advance_seed(device) -> None:
    """Once per training step (captured in the step's CUDA graph): new dropout masks next step."""
    seed_counter(device).add_(7919)


def next_salt() -> int:
    """Distinct per attention call site within a step (host-side, deterministic sequence)."""
    global _CALL_SALT
    _CALL_SALT = (_CALL_SALT * 1103515245 + 12345) & 0x7FFFFFFF
    return _CALL_SALT


def _row_strided(t: torch.Tensor):
    """(L, B, E) view whose (l, b) rows are `ld` elements apart (a slice of a wider projection) -> ld, else None"""
    l, b, e = t.shape
    if t.stride(2) == 1 and t.stride(0) == b * t.stride(1) and t.stride(1) >= e and t.stride(1) % 4 == 0:
        return t.stride(1)
    return None


def mask_bits(mask: torch.Tensor, batch: int):
    """Boolean / byte attention mask (True = not visible), (Lq, Lk) or (B, Lq, Lk) -> (bits_q, bits_k) for the fused
    kernels (include/coda_attention.h coda_attention_mask_pack): one 64-bit word per (row, 64-column tile)."""
    if mask.dim() == 2:
        mask = mask.unsqueeze(0)
    assert mask.dim() == 3 and mask.shape[0] in (1, batch), "attn_mask must be (Lq, Lk) or (B, Lq, Lk)"
    m = mask if mask.dtype == torch.uint8 else mask.to(torch.bool).view(torch.uint8) if mask.dtype == torch.bool \
        else (mask != 0).view(torch.uint8)
    _, lq, lk = m.shape
    sb = m.stride(0) if m.shape[0] == batch and batch > 1 else (0 if m.shape[0] == 1 else m.stride(0))
    bq = torch.empty((batch, lq, (lk + 63) // 64), dtype=torch.int64, device=m.device)
    bk = torch.empty((batch, lk, (lq + 63) // 64), dtype=torch.int64, device=m.device)
    with torch.cuda.device(m.device):
        st = lib().coda_attention_mask_pack(ctypes.c_int(batch), ctypes.c_int(lq), ctypes.c_int(lk), ptr(m),
                                            ctypes.c_longlong(sb), ctypes.c_longlong(m.stride(1)),
                                            ctypes.c_longlong(m.stride(2)), ptr(bq), ptr(bk), stream_of(m))
    check(st, "attention_mask_pack")
    return bq, bk


def radius_mask_bits(xyz: torch.Tensor, radius: float):
    """xyz (B, L, 3) fp32 -> bits (B, L, ceil(L/64)) int64 of the mask `cdist(xyz, xyz) >= radius` (reference
    models/transformer.py:155-162), packed on the device without the (B, L, L) distance matrix; symmetric, so the
    same tensor is both bits_q and bits_k."""
    b, l, _ = xyz.shape
    x = xyz.detach().float().contiguous()
    bits = torch.empty((b, l, (l + 63) // 64), dtype=torch.int64, device=x.device)
    with torch.cuda.device(x.device):
        st = lib().coda_attention_mask_radius(ctypes.c_int(b), ctypes.c_int(l), ptr(x), ctypes.c_float(float(radius)),
                                              ptr(bits), stream_of(x))
    check(st, "attention_mask_radius")
    return bits, bits


# operand planes of q / k / v in the forward of the fp32 attention: 2 = 16 mantissa bits, three cross products per
# contraction (3 = 24 bits, six).  Against the reference goldens (tests/test_model_gpu.py, all seven cases incl. the
# BASELINE-size and ScanNet-size ones) the forward's worst deviation does not change between 2 and 3 planes -- the
# attention operands are not what limits parity -- so the step runs on 2.  CODA_ATTN_NSPLIT=3 restores the wider split.
import os as _os
FORWARD_NSPLIT = int(_os.environ.get("CODA_ATTN_NSPLIT", "2"))


def forward(q, k, v, nhead: int, dropout_p: float = 0.0, salt: int = 0, nsplit: int | None = None, half_out: bool = False,
            mask=None):
    """q (Lq, B, E), k / v (Lk, B, E), fp32 or fp16 (all three alike), each either contiguous or a row-strided
    slice of a fused projection -> (out (Lq, B, E) fp32, lse (B*H, Lq)).  mask: (bits_q, bits_k) from mask_bits /
    radius_mask_bits, or None."""
    if nsplit is None:
        nsplit = FORWARD_NSPLIT
    lq, b, e = q.shape
    lk = k.shape[0]
    hd = e // nhead
    assert hd in (64, 128), "head dim must be 64 or 128"
    is_half = q.dtype == torch.float16
    assert k.dtype == q.dtype and v.dtype == q.dtype and q.dtype in (torch.float16, torch.float32)
    lds = [_row_strided(t) for t in (q, k, v)]
    if any(ld is None for ld in lds):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        lds = [e, e, e]
    half_out = bool(half_out) and lk <= 64 and hd == 64 and nsplit <= 2   # the single-tile instance only
    out = torch.empty((lq, b, e), dtype=torch.float16 if half_out else torch.float32, device=q.device)
    lse = torch.empty((b * nhead, lq), dtype=torch.float32, device=q.device)
    L = lib()
    L.coda_attention_workspace_bytes.restype = ctypes.c_longlong
    ws_bytes = L.coda_attention_workspace_bytes(b, nhead, lq, lk, hd, nsplit)
    ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device=q.device)
    seed_dev = seed_counter(q.device) if dropout_p > 0.0 else None
    ci, cl = ctypes.c_int, ctypes.c_longlong
    with torch.cuda.device(q.device):
        st = L.coda_attention_pack_strided(ci(b), ci(nhead), ci(lq), ci(lk), ci(hd), ci(nsplit),
                                           ctypes.c_float(float(hd) ** -0.5), ptr(q), ptr(k), ptr(v), cl(lds[0]),
                                           cl(lds[1]), cl(lds[2]), ci(1 if is_half else 0), ptr(ws), stream_of(q))
        check(st, "attention_pack")
        st = L.coda_attention_fwd_packed_masked(ci(b), ci(nhead), ci(lq), ci(lk), ci(hd), ci(nsplit), ptr(ws), ptr(out),
                                                ci(1 if half_out else 0), ptr(lse),
                                                ptr(None if mask is None else mask[0]), ctypes.c_float(dropout_p),
                                                ctypes.c_uint(salt & 0xFFFFFFFF), ptr(seed_dev), stream_of(q))
    check(st, "attention_fwd")
    return out, lse


def forward_half(q, k, v, nhead: int):
    """fp16 q / k / v (L <= 256, B, H * 64), contiguous or row-strided slices of a fused projection -> fp16 (L, B, E):
    the CLIP image tower's attention on half operands (include/coda_attention.h coda_attention_fwd_half).  Above 64
    tokens (ViT-B/16) the kernel reads q / k / v in place by TMA and needs no workspace."""
    l, b, e = q.shape
    assert q.dtype == k.dtype == v.dtype == torch.float16 and e // nhead == 64 and l <= 256 and k.shape[0] == l
    lds = [_row_strided(t) for t in (q, k, v)]
    if l > 64:   # TMA reads the slices in place: 16-byte aligned bases and row strides
        lds = [ld if ld is not None and ld % 8 == 0 and t.data_ptr() % 16 == 0 else None
               for ld, t in zip(lds, (q, k, v))]
    if any(ld is None for ld in lds):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        lds = [e, e, e]
    out = torch.empty((l, b, e), dtype=torch.float16, device=q.device)
    ws = None if l > 64 else torch.empty(3 * b * nhead * l * 64 * 2 + 512, dtype=torch.uint8, device=q.device)
    cl = ctypes.c_longlong
    with torch.cuda.device(q.device):
        st = lib().coda_attention_fwd_half(ctypes.c_int(b), ctypes.c_int(nhead), ctypes.c_int(l), ctypes.c_int(64), ptr(q),
                                           ptr(k), ptr(v), cl(lds[0]), cl(lds[1]), cl(lds[2]), ptr(out), ptr(ws),
                                           stream_of(q))
    check(st, "attention_fwd_half")
    return out


_LCG_A, _LCG_C = 747796405, 2891336453


def _lcg_jump():
    """(a[c], c[c]) with x_c = a[c] * s + c[c] (mod 2^32): the LCG stepped c + 1 times (attention_common.cuh)."""
    M = 0xFFFFFFFF
    a, c, ja, jc = _LCG_A, _LCG_C, [], []
    for _ in range(64):
        ja.append(a)
        jc.append(c)
        c = (c * _LCG_A + _LCG_C) & M
        a = (a * _LCG_A) & M
    return ja, jc


def dropout_keep(bh: int, lq: int, lk: int, dropout_p: float, salt: int, device, bh0: int = 0) -> torch.Tensor:
    """(bh, lq, lk) bool keep-mask of the (batch * head) rows bh0 .. bh0 + bh - 1, bit-identical to drop_keep() in
    csrc/attention_common.cuh."""
    M = 0xFFFFFFFF
    seed = (seed_counter(device).to(torch.int64) & M) + (salt & M)   # stays on the device: no sync
    ib = torch.arange(bh0, bh0 + bh, device=device, dtype=torch.int64).view(bh, 1, 1)
    iq = torch.arange(lq, device=device, dtype=torch.int64).view(1, lq, 1)
    ik = torch.arange(lk, device=device, dtype=torch.int64).view(1, 1, lk)
    h = (seed + ib * 0x9E3779B1 + iq * 0x85EBCA77 + (ik >> 6) * 0xC2B2AE3D) & M   # one hash per 64-key tile
    h = h ^ (h >> 15)
    h = (h * 0x2C1B3C6D) & M
    h = h ^ (h >> 12)
    h = (h * 0x297A2D39) & M
    h = h ^ (h >> 15)
    ja, jc = _lcg_jump()
    ja = torch.tensor(ja, dtype=torch.int64, device=device)[ik & 63]
    jc = torch.tensor(jc, dtype=torch.int64, device=device)[ik & 63]
    # 32 x 32 -> low 32 bits without overflowing int64: split the multiplier
    x = ((h * (ja & 0xFFFF)) + (((h * (ja >> 16)) & 0xFFFF) << 16) + jc) & M
    thresh = int(float(np.float32(dropout_p)) * 4294967296.0)
    return x >= thresh


def dropout_mult(bh: int, lq: int, lk: int, dropout_p: float, salt: int, device) -> torch.Tensor:
    """(bh, lq, lk) fp32 factor in {0, 1/(1-p)}: the dropout the forward kernel applied (one kernel)."""
    out = torch.empty((bh, lq, lk), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        st = lib().coda_attention_dropout_mult(ctypes.c_int(bh), ctypes.c_int(lq), ctypes.c_int(lk),
                                               ctypes.c_float(dropout_p), ctypes.c_uint(salt & 0xFFFFFFFF),
                                               ptr(seed_counter(device)), ptr(out),
                                               ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream))
    check(st, "attention_dropout_mult")
    return out


def backward(q, k, v, out, dout, lse, nhead: int, dropout_p: float = 0.0, salt: int = 0, mask=None, grads=None):
    """Fused wgmma backward (head dim 64 / 128): returns (dq, dk, dv), each shaped like its input.  q / k / v may
    be row-strided slices of a fused projection (read in place); `grads` = preallocated (dq, dk, dv) views, e.g. the
    slices of ONE packed gradient buffer of that projection (written in place, nothing to concatenate)."""
    lq, b, e = q.shape
    lk = k.shape[0]
    hd = e // nhead
    assert hd in (64, 128)
    lds = [_row_strided(t) for t in (q, k, v)]
    if any(ld is None for ld in lds) or any(t.data_ptr() % 16 for t in (q, k, v)):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        lds = [e, e, e]
    out, dout = out.contiguous(), dout.contiguous()
    if grads is None:
        grads = (torch.empty((lq, b, e), dtype=torch.float32, device=q.device),
                 torch.empty((lk, b, e), dtype=torch.float32, device=q.device),
                 torch.empty((lk, b, e), dtype=torch.float32, device=q.device))
    dq, dk, dv = grads
    ldg = [_row_strided(t) for t in grads]
    assert all(ld is not None for ld in ldg) and all(t.data_ptr() % 16 == 0 for t in grads)
    cl = ctypes.c_longlong
    L = lib()
    L.coda_attention_bwd_workspace_bytes.restype = ctypes.c_longlong
    ws = torch.empty(int(L.coda_attention_bwd_workspace_bytes(b, nhead, lq, lk, hd)), dtype=torch.uint8, device=q.device)
    seed_dev = seed_counter(q.device) if dropout_p > 0.0 else None
    with torch.cuda.device(q.device):
        st = L.coda_attention_bwd_ex(ctypes.c_int(b), ctypes.c_int(nhead), ctypes.c_int(lq), ctypes.c_int(lk),
                                     ctypes.c_int(hd), ctypes.c_float(float(hd) ** -0.5), ptr(q), ptr(k), ptr(v),
                                     cl(lds[0]), cl(lds[1]), cl(lds[2]), ptr(out), ptr(dout), ptr(lse), ptr(dq), ptr(dk),
                                     ptr(dv), cl(ldg[0]), cl(ldg[1]), cl(ldg[2]),
                                     ptr(None if mask is None else mask[0]), ptr(None if mask is None else mask[1]),
                                     ctypes.c_float(dropout_p), ctypes.c_uint(salt & 0xFFFFFFFF), ptr(seed_dev), ptr(ws),
                                     stream_of(q))
    check(st, "attention_bwd")
    return dq, dk, dv
