"""Fused multi-head attention on wgmma tensor cores (include/coda_attention.h).

forward : one launch per attention call; S = Q K^T, online softmax and O = P V are
          tiled through registers, the (Lq x Lk) probabilities never reach HBM.
backward: two wgmma kernels (dQ; dK / dV) that recompute P tile by tile from the saved
          log-sum-exp (csrc/attention_bwd_sm90.cu); nothing of size Lq x Lk is stored.
`_math` below is the plain-tensor formulation used by the tests as the numerics reference and by
the causal CLIP text tower, which runs once at model construction (never inside the step).
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from ._lib import check, lib, ptr, stream_of


def _math(q, k, v, nhead, dropout_p, training, causal, keep=None, attn_mask=None):
    """softmax(q k^T / sqrt(hd)) v per head in plain tensor ops: numerics reference in tests and the
    init-time CLIP text tower.  `keep` is an explicit (B*H, Lq, Lk) dropout keep-mask; `attn_mask` a boolean
    (B, Lq, Lk) mask (True = not visible)."""
    lq, b, e = q.shape
    lk = k.shape[0]
    hd = e // nhead
    qh = (q * (float(hd) ** -0.5)).reshape(lq, b * nhead, hd).transpose(0, 1)
    kh = k.reshape(lk, b * nhead, hd).transpose(0, 1)
    vh = v.reshape(lk, b * nhead, hd).transpose(0, 1)
    s = torch.bmm(qh, kh.transpose(1, 2))
    if causal:
        s = s + torch.full((lq, lk), float("-inf"), device=s.device, dtype=s.dtype).triu_(1)
    if attn_mask is not None:
        s = s.masked_fill(attn_mask.to(torch.bool).repeat_interleave(nhead, dim=0), float("-inf"))
    p = torch.softmax(s, dim=-1)
    if keep is not None:
        p = p * (keep if keep.dtype == p.dtype else keep.to(p.dtype) * (1.0 / (1.0 - float(np.float32(dropout_p)))))
    elif training and dropout_p > 0.0:
        p = torch.nn.functional.dropout(p, dropout_p)
    return torch.bmm(p, vh).transpose(0, 1).reshape(lq, b, e)


def kernel_available() -> bool:
    return hasattr(lib(), "coda_attention_fwd")


class _Attention(torch.autograd.Function):
    """layout "q_k_v": three separate projections.  "qkv": `a` is ONE fused (L, B, 3E) projection (encoder
    self-attention); "qk_v": `a` = fused (L, B, 2E) q|k projection, `b` = v (decoder self-attention).  The fused
    forms read their slices in place and the backward writes dq / dk (/ dv) into one packed gradient tensor: the
    gradient of the fused projection needs no concatenation and arrives contiguous at its weight-gradient GEMM."""

    @staticmethod
    def forward(ctx, a, b, c, layout, nhead, dropout_p, salt, mask):
        from . import attention_launch

        if layout == "qkv":
            e = a.shape[-1] // 3
            q, k, v = a[..., :e], a[..., e: 2 * e], a[..., 2 * e:]
        elif layout == "qk_v":
            e = a.shape[-1] // 2
            q, k, v = a[..., :e], a[..., e:], b
        else:
            q, k, v = a, b, c
        out, lse = attention_launch.forward(q, k, v, nhead, dropout_p, salt, mask=mask)
        ctx.save_for_backward(a, b, c, out, lse)
        ctx.layout, ctx.nhead, ctx.dropout_p, ctx.salt, ctx.mask = layout, nhead, dropout_p, salt, mask
        return out

    @staticmethod
    def backward(ctx, dout):
        from . import attention_launch

        a, b, c, out, lse = ctx.saved_tensors
        # fused wgmma backward (dQ kernel + dK/dV kernel); P is recomputed tile by tile, never stored
        kw = dict(mask=ctx.mask)
        if ctx.layout == "qkv":
            e = a.shape[-1] // 3
            da = torch.empty(a.shape, dtype=torch.float32, device=a.device)
            attention_launch.backward(a[..., :e], a[..., e: 2 * e], a[..., 2 * e:], out, dout, lse, ctx.nhead,
                                      ctx.dropout_p, ctx.salt, grads=(da[..., :e], da[..., e: 2 * e], da[..., 2 * e:]), **kw)
            return da, None, None, None, None, None, None, None
        if ctx.layout == "qk_v":
            e = a.shape[-1] // 2
            da = torch.empty(a.shape, dtype=torch.float32, device=a.device)
            db = torch.empty(b.shape, dtype=torch.float32, device=a.device)
            attention_launch.backward(a[..., :e], a[..., e:], b, out, dout, lse, ctx.nhead, ctx.dropout_p, ctx.salt,
                                      grads=(da[..., :e], da[..., e:], db), **kw)
            return da, db, None, None, None, None, None, None
        dq, dk, dv = attention_launch.backward(a, b, c, out, dout, lse, ctx.nhead, ctx.dropout_p, ctx.salt, **kw)
        return dq, dk, dv, None, None, None, None, None


def attention(q, k, v, nhead, dropout_p=0.0, training=False, causal=False, mask=None):
    """q (Lq, B, E), k / v (Lk, B, E) -> (Lq, B, E); see ops.attention.  mask: packed (bits_q, bits_k)."""
    if not q.is_cuda:
        raise RuntimeError("attention: CPU not supported")
    hd = q.shape[-1] // nhead
    if causal or q.dtype != torch.float32 or hd not in (64, 128):
        # CLIP text tower only (causal, fp16/fp32, runs ONCE at model construction, never inside the step)
        if mask is not None:
            raise NotImplementedError("attention masks exist on the fp32 head-dim 64 / 128 kernels only")
        return _math(q, k, v, nhead, dropout_p, training, causal)
    from . import attention_launch

    p = float(dropout_p) if training else 0.0
    return _Attention.apply(q, k, v, "q_k_v", nhead, p, attention_launch.next_salt() if p > 0.0 else 0, mask)


def attention_fused(a, b, layout, nhead, dropout_p=0.0, training=False, mask=None):
    """Self-attention on fused projections: layout "qkv" (a = (L, B, 3E)) or "qk_v" (a = (L, B, 2E) q|k, b = v)."""
    if not a.is_cuda:
        raise RuntimeError("attention: CPU not supported")
    e = a.shape[-1] // (3 if layout == "qkv" else 2)
    if a.dtype != torch.float32 or (e // nhead) not in (64, 128):
        # head dims the wgmma kernels do not cover (reduced test configurations): the three-tensor entry decides
        return attention(a[..., :e], a[..., e: 2 * e], a[..., 2 * e:] if layout == "qkv" else b, nhead, dropout_p,
                         training, False, mask)
    from . import attention_launch

    p = float(dropout_p) if training else 0.0
    return _Attention.apply(a, b, None, layout, nhead, p, attention_launch.next_salt() if p > 0.0 else 0, mask)
