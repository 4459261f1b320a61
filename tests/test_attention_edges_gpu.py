"""Every wgmma attention instance against a float64 reference, at the edges where the kernels' tile walk changes.

tests/attention_instances.py restates which kernel instance, ring depth and tile walk a shape gets;
tests/test_attention_instances_cpu.py checks that the case lists below (with those of test_attention_gpu.py) run
every instance in every variant, every tail and every ring wrap.  The reference is attention_sm100._math in float64,
with the dropout keep-mask rebuilt by attention_launch.dropout_keep and the boolean mask the kernels get packed.

Besides the aggregate comparisons, the pattern tests make each kernel write P o M itself, through one-hot operands,
so that the set of exact zeros it produces can be compared with the twin's mask element by element.

The bars and the worst errors measured against them are listed with FWD_TOL.
"""
import ctypes

import numpy as np
import pytest
import torch

from coda_neurips2023_b200 import attention_launch, attention_sm100
from coda_neurips2023_b200._lib import CodaError, lib, ptr, stream_of

pytestmark = pytest.mark.gpu

P_DROP = 0.1
VARIANTS = ("plain", "mask", "dropout", "mask+dropout")
# Each bar is at least 3x the worst error its checks measured (in brackets), H100 80GB HBM3 at a 700 W power limit.
# output, relative to the largest output, per forward operand-plane count [6.5e-3, 2.1e-5, 2.4e-6]
FWD_TOL = {1: 2e-2, 2: 1e-4, 3: 1e-5}
# log-sum-exp, absolute (natural-log units), per forward operand-plane count [7.8e-3, 2.2e-5, 1.0e-5]
LSE_TOL = {1: 3e-2, 2: 1e-4, 3: 5e-5}
# gradients, relative to the largest gradient of the same tensor: the backward runs on two planes [dq 6.3e-5 at the
# designed edges, 3.5e-5 elsewhere; dk 2.7e-5; dv 2.3e-5]
GRAD_TOL = 2e-4
# P o M / (1 - p) read out through one-hot operands, relative to its largest element: forward per plane count (P
# itself carries at most two planes) [2.6e-3, 5.5e-6, 4.0e-6], and the dK/dV and dQ kernels [6.6e-6, 7.8e-6]
PATTERN_TOL = {1: 1e-2, 2: 2.5e-5, 3: 1.5e-5}
PATTERN_BWD_TOL = 3e-5


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


@pytest.fixture
def seed_at():
    """sets the device-side dropout step counter and restores it afterwards: other tests keep their streams"""
    ctr = attention_launch.seed_counter(torch.device("cuda", torch.cuda.current_device()))
    saved = ctr.clone()
    yield lambda value: ctr.fill_(value)
    ctr.copy_(saved)


def _check(what, err, bar):
    assert err < bar, f"{what}: {err:.3e} (bar {bar:.1e})"


def _rel(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


def _heads(x, h):
    """(L, B, H * hd) -> (B * H, L, hd) float64"""
    l, b, e = x.shape
    return x.double().reshape(l, b * h, e // h).transpose(0, 1)


def _scores64(q, k, h, mask=None):
    hd = q.shape[-1] // h
    s = _heads(q, h) @ _heads(k, h).transpose(1, 2) * hd ** -0.5
    return s if mask is None else s.masked_fill(mask.repeat_interleave(h, dim=0), float("-inf"))


def _keep_scale(p):
    return 1.0 / (1.0 - float(np.float32(p)))


def _random_mask(b, lq, lk, density, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mask = torch.rand(b, lq, lk, device="cuda", generator=g) < density
    mask[:, : lq // 2, : min(lk, 192) // 2] = True      # leading key tiles fully masked for half the rows
    mask[:, :, lk - 1] = False                          # every row keeps at least one key
    return mask


def _qkv(lq, lk, b, e, seed, qk_scale=1.2):
    torch.manual_seed(seed)
    return (torch.randn(lq, b, e, device="cuda") * qk_scale, torch.randn(lk, b, e, device="cuda") * qk_scale,
            torch.randn(lk, b, e, device="cuda"))


def _bwd_ref(q, k, v, g, h, p, keep, mask):
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref = attention_sm100._math(q64, k64, v64, h, p, False, False, keep, attn_mask=mask)
    return ref.detach(), torch.autograd.grad(ref, (q64, k64, v64), g.double())


# ------------------------------------------------------------------ every forward instance x variant
# (hd, warpgroups) -> (lq, lk): one key tile, a key tail, rings that wrap once and twice, and (two warpgroups) a
# query tail in each warpgroup of the last CTA; tests/attention_instances.py says which shape does what
FWD_SHAPES = {
    (64, 1): [(64, 64), (37, 100), (64, 300), (5, 600)],
    (64, 2): [(130, 50), (200, 100), (65, 200), (192, 300), (128, 600)],
    (128, 1): [(64, 50), (100, 100), (130, 200), (1, 300), (70, 600)],
}
FWD_CASES = [(lq, lk, hd, ns, var) for (hd, _), shapes in FWD_SHAPES.items() for lq, lk in shapes
             for ns in (1, 2, 3) for var in VARIANTS]


@pytest.mark.parametrize("lq,lk,hd,nsplit,variant", FWD_CASES)
def test_forward_instance_vs_fp64(lq, lk, hd, nsplit, variant, seed_at):
    b, h = 2, 2
    q, k, v = _qkv(lq, lk, b, h * hd, lq * 7 + lk + nsplit)
    mask = _random_mask(b, lq, lk, 0.5, lq + lk) if "mask" in variant else None
    p = P_DROP if "dropout" in variant else 0.0
    seed_at(1000 + lk)
    salt = 31 * lq + nsplit
    out, lse = attention_launch.forward(q, k, v, h, dropout_p=p, salt=salt, nsplit=nsplit,
                                        mask=None if mask is None else attention_launch.mask_bits(mask, b))
    keep = attention_launch.dropout_keep(b * h, lq, lk, p, salt, q.device) if p else None
    ref = attention_sm100._math(q.double(), k.double(), v.double(), h, p, False, False, keep, attn_mask=mask)
    _check(f"forward out, {nsplit} planes", _rel(out, ref), FWD_TOL[nsplit])
    ref_lse = torch.logsumexp(_scores64(q, k, h, mask), dim=-1)
    _check(f"forward lse, {nsplit} planes", (lse.double() - ref_lse).abs().max().item(), LSE_TOL[nsplit])


# ------------------------------------------------------------------ both backward instances x variant
# hd -> (lq, lk): rings of the dQ (over keys) and dK/dV (over queries) kernels that wrap twice, Lq < 64, Lk < 64,
# and query / key tails in each warpgroup of a two-warpgroup CTA
BWD_SHAPES = {
    64: [(600, 600), (37, 130), (200, 37), (130, 100)],
    128: [(330, 330), (37, 130), (200, 37), (100, 70)],
}
BWD_CASES = [(lq, lk, hd, var) for hd, shapes in BWD_SHAPES.items() for lq, lk in shapes for var in VARIANTS]


@pytest.mark.parametrize("lq,lk,hd,variant", BWD_CASES)
def test_backward_instance_vs_fp64(lq, lk, hd, variant, seed_at):
    b, h = 2, 2
    q, k, v = _qkv(lq, lk, b, h * hd, lq + 3 * lk)
    mask = _random_mask(b, lq, lk, 0.5, lq * lk) if "mask" in variant else None
    bits = None if mask is None else attention_launch.mask_bits(mask, b)
    p = P_DROP if "dropout" in variant else 0.0
    seed_at(77 + lq)
    salt = 5 + lk
    out, lse = attention_launch.forward(q, k, v, h, dropout_p=p, salt=salt, nsplit=3, mask=bits)
    g = torch.randn_like(out)
    got = attention_launch.backward(q, k, v, out, g, lse, h, p, salt, mask=bits)
    keep = attention_launch.dropout_keep(b * h, lq, lk, p, salt, q.device) if p else None
    _, exp = _bwd_ref(q, k, v, g, h, p, keep, mask)
    for name, a, e in zip(("dq", "dk", "dv"), got, exp):
        _check(f"backward {name}", _rel(a, e), GRAD_TOL)


# ------------------------------------------------------------------ the step's forward -> backward chain
# tools/bench_attention.py BWD_CASES, through the entry each call site of models/transformer.py uses:
# name, layout, b, h, lq, lk, hd
CHAIN_CASES = [
    ("encoder self", "qkv", 8, 4, 2048, 2048, 64),
    ("decoder cross", "q_k_v", 8, 4, 256, 2048, 128),
    ("decoder self", "qk_v", 8, 4, 256, 256, 128),
]


@pytest.mark.parametrize("name,layout,b,h,lq,lk,hd", CHAIN_CASES)
def test_step_chain_vs_fp64(name, layout, b, h, lq, lk, hd, seed_at, monkeypatch):
    """The step's forward (attention_launch.FORWARD_NSPLIT planes, dropout 0.1) hands its lse to the backward.  The
    reference is built one (batch, head) at a time: the whole problem in float64 would take gigabytes."""
    e = h * hd
    torch.manual_seed(lq + lk + hd)
    salt = 4321
    monkeypatch.setattr(attention_launch, "next_salt", lambda: salt)
    seed_at(9001)
    if layout == "qkv":
        a = (torch.randn(lq, b, 3 * e, device="cuda") * 1.2).requires_grad_(True)
        leaves = (a,)
        out = attention_sm100.attention_fused(a, None, "qkv", h, P_DROP, True)
        q, k, v = a.detach().split(e, dim=-1)
    elif layout == "qk_v":
        a = (torch.randn(lq, b, 2 * e, device="cuda") * 1.2).requires_grad_(True)
        vs = torch.randn(lk, b, e, device="cuda", requires_grad=True)
        leaves = (a, vs)
        out = attention_sm100.attention_fused(a, vs, "qk_v", h, P_DROP, True)
        (q, k), v = a.detach().split(e, dim=-1), vs.detach()
    else:
        q = (torch.randn(lq, b, e, device="cuda") * 1.2).requires_grad_(True)
        k = (torch.randn(lk, b, e, device="cuda") * 1.2).requires_grad_(True)
        v = torch.randn(lk, b, e, device="cuda", requires_grad=True)
        leaves = (q, k, v)
        out = attention_sm100.attention(q, k, v, h, P_DROP, True)
        q, k, v = q.detach(), k.detach(), v.detach()
    g = torch.randn_like(out)
    grads = torch.autograd.grad(out, leaves, g)
    got = {"out": out.detach()}
    if layout == "q_k_v":
        got["dq"], got["dk"], got["dv"] = grads
    else:
        got["dq"], got["dk"] = grads[0][..., :e], grads[0][..., e: 2 * e]
        got["dv"] = grads[0][..., 2 * e:] if layout == "qkv" else grads[1]
    diff, peak = dict.fromkeys(got, 0.0), dict.fromkeys(got, 0.0)
    scale, m = hd ** -0.5, _keep_scale(P_DROP)
    for i in range(b * h):
        bi, hi = divmod(i, h)
        cols = slice(hi * hd, (hi + 1) * hd)
        qh, kh, vh, gh = (t[:, bi, cols].double() for t in (q, k, v, g))
        keep = attention_launch.dropout_keep(1, lq, lk, P_DROP, salt, q.device, bh0=i)[0].double() * m
        pr = torch.softmax((qh * scale) @ kh.T, dim=-1)
        pt = pr * keep
        o = pt @ vh
        ds = pr * ((gh @ vh.T) * keep - (gh * o).sum(-1, keepdim=True))
        ref = {"out": o, "dq": scale * ds @ kh, "dk": scale * ds.T @ qh, "dv": pt.T @ gh}
        for key, r in ref.items():
            diff[key] = max(diff[key], (got[key][:, bi, cols].double() - r).abs().max().item())
            peak[key] = max(peak[key], r.abs().max().item())
    _check(f"{name} chain out", diff["out"] / peak["out"], FWD_TOL[attention_launch.FORWARD_NSPLIT])
    for key in ("dq", "dk", "dv"):
        _check(f"{name} chain {key}", diff[key] / peak[key], GRAD_TOL)


# ------------------------------------------------------------------ element-exact dropout and mask patterns
PATTERN_VARIANTS = ("mask", "dropout", "mask+dropout")
# forward: (hd, warpgroups) -> (lq, lk); every key position 0, 63, 64 and the last of a tail tile is read out
PATTERN_FWD_SHAPES = {(64, 1): (64, 600), (64, 2): (200, 600), (128, 1): (130, 300)}
PATTERN_FWD_CASES = [(lq, lk, hd, ns, var) for (hd, _), (lq, lk) in PATTERN_FWD_SHAPES.items() for ns in (1, 2, 3)
                     for var in PATTERN_VARIANTS]
# backward: hd -> (lq, lk) of the dK/dV read-out (dV through an identity block of dO over queries) and of the dQ
# read-out (dQ through an identity block of K over keys)
PATTERN_DKV_SHAPES = {64: (300, 200), 128: (260, 200)}
PATTERN_DQ_SHAPES = {64: (200, 200), 128: (100, 300)}
PATTERN_BWD_CASES = [(hd, var) for hd in (64, 128) for var in PATTERN_VARIANTS]


def _pattern_setup(variant, b, h, lq, lk, seed):
    mask = _random_mask(b, lq, lk, 0.3, seed) if "mask" in variant else None
    p = P_DROP if "dropout" in variant else 0.0
    return mask, p, None if mask is None else attention_launch.mask_bits(mask, b)


def _expected_zeros(keep, mask, h):
    """where P o M is exactly zero: dropped or masked"""
    dead = None if keep is None else ~keep
    if mask is not None:
        m = mask.repeat_interleave(h, dim=0)
        dead = m if dead is None else dead | m
    return dead


def _block(rows, b, h, hd, c0, n):
    """(rows, B, H * hd) with x[c0 + d, :, head * hd + d] = 1 for d < n, in every head"""
    x = torch.zeros(rows, b, h, hd, device="cuda")
    d = torch.arange(n, device="cuda")
    x[c0 + d, :, :, d] = 1.0
    return x.reshape(rows, b, h * hd)


def _per_head(x, h):
    """(L, B, H * hd) -> (B * H, L, hd)"""
    l, b, e = x.shape
    return x.reshape(l, b, h, e // h).permute(1, 2, 0, 3).reshape(b * h, l, e // h)


@pytest.mark.parametrize("lq,lk,hd,nsplit,variant", PATTERN_FWD_CASES)
def test_forward_writes_the_twins_dropout_and_mask_pattern(lq, lk, hd, nsplit, variant, seed_at):
    """V = an identity block over keys [c0, c0 + hd) makes out[q, d] = P[q, c0 + d] M[q, c0 + d] / (1 - p): the
    forward's own dropout and mask decisions, key by key.  Scores stay small (|s| < 20), so no kept P underflows."""
    b, h = 2, 2
    q, k, _ = _qkv(lq, lk, b, h * hd, 11 * lq + lk + nsplit, qk_scale=0.5)
    mask, p, bits = _pattern_setup(variant, b, h, lq, lk, lq + nsplit)
    seed_at(300 + nsplit)
    salt = 17 * nsplit + lq
    got = torch.empty(b * h, lq, lk, device="cuda")
    for c0 in range(0, lk, hd):
        n = min(hd, lk - c0)
        out, _ = attention_launch.forward(q, k, _block(lk, b, h, hd, c0, n), h, dropout_p=p, salt=salt, nsplit=nsplit,
                                          mask=bits)
        got[:, :, c0: c0 + n] = _per_head(out, h)[..., :n]
    keep = attention_launch.dropout_keep(b * h, lq, lk, p, salt, q.device) if p else None
    s = _scores64(q, k, h, mask)
    assert s.abs()[torch.isfinite(s)].max().item() < 20
    ref = torch.softmax(s, dim=-1) * (keep.double() * _keep_scale(p) if keep is not None else 1.0)
    assert torch.equal(got == 0, _expected_zeros(keep, mask, h))
    _check(f"forward pattern, {nsplit} planes", _rel(got, ref), PATTERN_TOL[nsplit])


def _pattern_bwd_ref(q, k, lse, h, keep, mask, p):
    """P~ = exp(s - lse) M / (1 - p) with the lse the backward was given: the backward kernels' own P"""
    pr = torch.exp(_scores64(q, k, h, mask) - lse.double().unsqueeze(-1))
    return pr * (keep.double() * _keep_scale(p)) if keep is not None else pr


@pytest.mark.parametrize("hd,variant", PATTERN_BWD_CASES)
def test_dkv_kernel_writes_the_twins_dropout_and_mask_pattern(hd, variant, seed_at):
    """dO = an identity block over queries [c0, c0 + hd) makes dV[k, d] = P~[c0 + d, k]: the dK/dV kernel's dropout
    (hashed per query column, ktile and key position in the tile) and mask decisions, element by element."""
    b, h = 2, 2
    lq, lk = PATTERN_DKV_SHAPES[hd]
    q, k, v = _qkv(lq, lk, b, h * hd, hd + lq, qk_scale=0.5)
    mask, p, bits = _pattern_setup(variant, b, h, lq, lk, hd + 1)
    seed_at(4000 + hd)
    salt = 23 + hd
    out, lse = attention_launch.forward(q, k, v, h, dropout_p=p, salt=salt, nsplit=3, mask=bits)
    got = torch.empty(b * h, lq, lk, device="cuda")
    for c0 in range(0, lq, hd):
        n = min(hd, lq - c0)
        _, _, dv = attention_launch.backward(q, k, v, out, _block(lq, b, h, hd, c0, n), lse, h, p, salt, mask=bits)
        got[:, c0: c0 + n, :] = _per_head(dv, h)[..., :n].transpose(1, 2)
    keep = attention_launch.dropout_keep(b * h, lq, lk, p, salt, q.device) if p else None
    ref = _pattern_bwd_ref(q, k, lse, h, keep, mask, p)
    assert torch.equal(got == 0, _expected_zeros(keep, mask, h))
    _check("dK/dV pattern", _rel(got, ref), PATTERN_BWD_TOL)


@pytest.mark.parametrize("hd,variant", PATTERN_BWD_CASES)
def test_dq_kernel_writes_the_twins_dropout_and_mask_pattern(hd, variant, seed_at):
    """out = 0 makes D = 0; V = ones and dO = e_0 make dP = 1; K = an identity block over keys [c0, c0 + hd) then
    gives dQ[q, d] = scale P[q, c0 + d] M[q, c0 + d] / (1 - p): the dQ kernel's own decisions, key by key."""
    b, h = 2, 2
    lq, lk = PATTERN_DQ_SHAPES[hd]
    e = h * hd
    torch.manual_seed(hd + 5)
    q = torch.randn(lq, b, e, device="cuda") * 2.0
    v = torch.ones(lk, b, e, device="cuda")
    dout = torch.zeros(lq, b, h, hd, device="cuda")
    dout[..., 0] = 1.0
    dout = dout.reshape(lq, b, e)
    mask, p, bits = _pattern_setup(variant, b, h, lq, lk, hd + 2)
    seed_at(5000 + hd)
    salt = 29 + hd
    got = torch.empty(b * h, lq, lk, device="cuda")
    ref = torch.empty(b * h, lq, lk, device="cuda", dtype=torch.float64)
    keep = attention_launch.dropout_keep(b * h, lq, lk, p, salt, q.device) if p else None
    for c0 in range(0, lk, hd):
        n = min(hd, lk - c0)
        k = _block(lk, b, h, hd, c0, n)
        out, lse = attention_launch.forward(q, k, v, h, dropout_p=p, salt=salt, nsplit=3, mask=bits)
        dq, _, _ = attention_launch.backward(q, k, v, torch.zeros_like(out), dout, lse, h, p, salt, mask=bits)
        got[:, :, c0: c0 + n] = _per_head(dq, h)[..., :n]
        ref[:, :, c0: c0 + n] = _pattern_bwd_ref(q, k, lse, h, keep, mask, p)[..., c0: c0 + n] * hd ** -0.5
    assert torch.equal(got == 0, _expected_zeros(keep, mask, h))
    _check("dQ pattern", _rel(got, ref), PATTERN_BWD_TOL)


# ------------------------------------------------------------------ designed softmax edges
EDGE_CASES = [(64, 40), (64, 200), (128, 130)]      # hd, lq: hd-64 one- and two-warpgroup CTAs, hd 128


@pytest.mark.parametrize("p", [0.0, P_DROP])
@pytest.mark.parametrize("hd,lq", EDGE_CASES)
def test_designed_softmax_edges(hd, lq, p, seed_at):
    """Each row's maximum arrives in the last (tail) key tile, 30 above every earlier score (the running output and
    sum are rescaled by about 2^-43); three rows see only the last key of that tail tile; five keys are visible to no query,
    so their dK and dV are exactly 0."""
    b, h, lk = 2, 2, 300
    e = h * hd
    q, k, v = _qkv(lq, lk, b, e, hd + lq, qk_scale=0.3)
    lonely = [0, lq // 2, lq - 1]
    # the jump of 30 sits on a component of Q: dQ = scale dS K sums dS over the tail keys, where it cancels, so a large
    # K component would scale the rounding of dP and dS against a small result; dK carries the factor in its value
    tail0 = (lk - 1) // 64 * 64
    q.view(lq, b, h, hd)[..., 0] = 120.0 * hd ** 0.5
    q.view(lq, b, h, hd)[lonely, :, :, 0] = 0.0
    k.view(lk, b, h, hd)[..., 0] = 0.0
    k.view(lk, b, h, hd)[tail0:, :, :, 0] = 0.25
    mask = torch.zeros(b, lq, lk, dtype=torch.bool, device="cuda")
    dead = [0, 63, 64, 150, lk - 2]
    mask[:, :, dead] = True
    mask[:, lonely, :] = True
    mask[:, lonely, lk - 1] = False
    bits = attention_launch.mask_bits(mask, b)
    seed_at(61)
    salt = 3 + hd
    keep = attention_launch.dropout_keep(b * h, lq, lk, p, salt, q.device) if p else None
    g = torch.randn(lq, b, e, device="cuda")
    ref, (rq, rk, rv) = _bwd_ref(q, k, v, g, h, p, keep, mask)
    ref_lse = torch.logsumexp(_scores64(q, k, h, mask), dim=-1)
    assert (ref_lse[:, lonely] - _scores64(q, k, h)[:, lonely, lk - 1]).abs().max() < 1e-12
    for ns in (2, 3):       # the backward below runs on the three-plane forward's out and lse
        out, lse = attention_launch.forward(q, k, v, h, dropout_p=p, salt=salt, nsplit=ns, mask=bits)
        _check(f"edges forward out, {ns} planes", _rel(out, ref), FWD_TOL[ns])
        _check(f"edges forward lse, {ns} planes", (lse.double() - ref_lse).abs().max().item(), LSE_TOL[ns])
    dq, dk, dv = attention_launch.backward(q, k, v, out, g, lse, h, p, salt, mask=bits)
    for name, a, r in (("dq", dq, rq), ("dk", dk, rk), ("dv", dv, rv)):
        _check(f"edges backward {name}", _rel(a, r), GRAD_TOL)
    assert torch.all(dk[dead] == 0) and torch.all(dv[dead] == 0)


# ------------------------------------------------------------------ determinism
@pytest.mark.parametrize("hd,lq,lk", [(64, 1000, 1000), (64, 50, 700), (128, 256, 1000)])
def test_same_bits_twice(hd, lq, lk, seed_at):
    """No atomics in the forward, dQ or dK/dV kernels: a repeated call, after a different launch in between, returns
    the same bits."""
    b, h = 2, 4
    q, k, v = _qkv(lq, lk, b, h * hd, 8 * hd + lk)
    bits = attention_launch.mask_bits(_random_mask(b, lq, lk, 0.3, 9), b)
    seed_at(12)
    g = torch.randn(lq, b, h * hd, device="cuda")
    runs = []
    for _ in range(2):
        out, lse = attention_launch.forward(q, k, v, h, dropout_p=P_DROP, salt=8, mask=bits)
        runs.append((out, lse, *attention_launch.backward(q, k, v, out, g, lse, h, P_DROP, 8, mask=bits)))
        ox, lx = attention_launch.forward(k[:77], q, q, h)           # another shape, grid and ring walk
        attention_launch.backward(k[:77], q, q, ox, ox, lx, h)
    for a, c in zip(*runs):
        assert torch.equal(a, c)


# ------------------------------------------------------------------ the fp16 instance and fp16 output
HALF_CASES = [1, 37, 64]                            # l of coda_attention_fwd_half (the CLIP image tower's 50)
HALF_OUT_CASES = [(37, 64, 1), (37, 64, 2), (200, 50, 1), (200, 50, 2)]     # lq, lk, nsplit


@pytest.mark.parametrize("l", HALF_CASES)
def test_half_operand_instance_vs_fp64(l):
    torch.manual_seed(l)
    b, h = 3, 4
    q, k, v = ((torch.randn(l, b, h * 64, device="cuda") * 0.8).half() for _ in range(3))
    out = attention_launch.forward_half(q, k, v, h)
    ref = attention_sm100._math(q.double(), k.double(), v.double(), h, 0.0, False, False)
    _check("fp16 instance", _rel(out, ref), 2e-3)


@pytest.mark.parametrize("lq,lk,nsplit", HALF_OUT_CASES)
def test_half_out_is_the_fp32_result_rounded_once(lq, lk, nsplit):
    q, k, v = _qkv(lq, lk, 2, 4 * 64, lq + lk)
    out16, lse16 = attention_launch.forward(q, k, v, 4, nsplit=nsplit, half_out=True)
    out32, lse32 = attention_launch.forward(q, k, v, 4, nsplit=nsplit)
    assert out16.dtype == torch.float16 and torch.equal(out16, out32.half()) and torch.equal(lse16, lse32)


# ------------------------------------------------------------------ contract
def test_half_out_with_a_mask_is_rejected():
    """fp16 output exists for the unmasked single key tile only: with a mask the C entry returns CODA_EINVAL"""
    lq = lk = 50
    b, h, hd = 2, 2, 64
    q, k, v = _qkv(lq, lk, b, h * hd, 1)
    bits = attention_launch.mask_bits(_random_mask(b, lq, lk, 0.3, 1), b)
    L = lib()
    L.coda_attention_workspace_bytes.restype = ctypes.c_longlong
    ws = torch.empty(int(L.coda_attention_workspace_bytes(b, h, lq, lk, hd, 2)), dtype=torch.uint8, device="cuda")
    out = torch.empty(lq, b, h * hd, dtype=torch.float16, device="cuda")
    lse = torch.empty(b * h, lq, device="cuda")
    ci = ctypes.c_int
    assert L.coda_attention_pack(ci(b), ci(h), ci(lq), ci(lk), ci(hd), ci(2), ctypes.c_float(hd ** -0.5), ptr(q),
                                 ptr(k), ptr(v), ptr(ws), stream_of(q)) == 0
    call = lambda m: L.coda_attention_fwd_packed_masked(  # noqa: E731
        ci(b), ci(h), ci(lq), ci(lk), ci(hd), ci(2), ptr(ws), ptr(out), ci(1), ptr(lse), ptr(m), ctypes.c_float(0.0),
        ctypes.c_uint(0), ptr(None), stream_of(q))
    assert call(bits[0]) == -1          # CODA_EINVAL
    assert call(None) == 0
    with pytest.raises(CodaError, match="attention_fwd failed"):
        attention_launch.forward(q, k, v, h, nsplit=2, half_out=True, mask=bits)


@pytest.mark.parametrize("hd,lq,lk", [(64, 130, 200), (128, 100, 70)])
def test_gradient_views_leave_the_rest_of_their_buffer_untouched(hd, lq, lk, seed_at):
    """`grads=` views whose rows are ld > E apart, inside sentinel-filled buffers: the views get the bits of a call
    with fresh tensors and every column outside them keeps the sentinel."""
    b, h = 2, 2
    e = h * hd
    q, k, v = _qkv(lq, lk, b, e, hd + lk)
    bits = attention_launch.mask_bits(_random_mask(b, lq, lk, 0.3, 3), b)
    seed_at(31)
    out, lse = attention_launch.forward(q, k, v, h, dropout_p=P_DROP, salt=2, mask=bits)
    g = torch.randn_like(out)
    want = attention_launch.backward(q, k, v, out, g, lse, h, P_DROP, 2, mask=bits)
    sentinel = -1234.5
    bq = torch.full((lq, b, e + 8), sentinel, device="cuda")
    bkv = torch.full((lk, b, 2 * e + 12), sentinel, device="cuda")
    views = (bq[..., 4: 4 + e], bkv[..., 4: 4 + e], bkv[..., e + 8: 2 * e + 8])
    attention_launch.backward(q, k, v, out, g, lse, h, P_DROP, 2, mask=bits, grads=views)
    for a, c in zip(views, want):
        assert torch.equal(a, c)
    assert (bq[..., :4] == sentinel).all() and (bq[..., 4 + e:] == sentinel).all()
    assert (bkv[..., :4] == sentinel).all() and (bkv[..., 4 + e: e + 8] == sentinel).all()
    assert (bkv[..., 2 * e + 8:] == sentinel).all()
