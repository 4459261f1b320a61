"""The step's glue kernels against fp64 at every instance and edge, and their dropout masks element by element.

Covers the LayerNorm family of csrc/detr_kernels.cu (every NV instance of the plain, `+ pos`, row-mapped, fp16 and
joined forms), everything in csrc/step_kernels.cu (BatchNorm on rows, dropout, clip + AdamW, n-ary sum, masked L1),
row softmax and the Hungarian matcher.  The C entry points are called through `lib()` where the `ops` wrappers cannot
reach an edge (explicit seeds and salts, AdamW chunks at unaligned offsets, row-mapped LayerNorm into a sentinel-filled
buffer).  tests/step_glue_paths.py restates which instance and path each case runs, and
tests/test_step_glue_paths_cpu.py checks, without a GPU, that the case lists below reach all of them.
"""
import ctypes

import numpy as np
import pytest
import torch

import step_glue_paths as P

pytestmark = pytest.mark.gpu

_i, _ll, _f, _u = ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_uint
PS = (1e-3, 0.1, 0.5, 0.9)   # dropout rates every masked kernel runs at
EPS = 1e-5
WORST: dict = {}             # check -> worst error seen in this session


def _bar(name, err, bar):
    err = float(err)
    WORST[name] = max(WORST.get(name, 0.0), err)
    assert err <= bar, f"{name}: {err:.3e} > {bar:.1e}"


def _rel(got, exp):
    """max |got - exp| over the largest |exp|"""
    exp = exp.double()
    return ((got.double() - exp).abs().max() / exp.abs().max().clamp_min(1e-300)).item()


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _L():
    from coda_neurips2023_b200._lib import lib

    L = lib()
    L.coda_layer_norm_bwd_scratch.restype = ctypes.c_longlong
    L.coda_grad_norm_scratch_floats.restype = ctypes.c_longlong
    return L


def _ok(status, what):
    from coda_neurips2023_b200._lib import check

    check(status, what)


def _p(t):
    from coda_neurips2023_b200._lib import ptr

    return ptr(t)


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bits(t):
    return t.view(torch.int32)


def _seed_tensor(seed):
    s = seed & 0xFFFFFFFF
    return torch.tensor([s - (1 << 32) if s >= 1 << 31 else s], dtype=torch.int32, device="cuda")


def _keep(seed, salt, p, n):
    return torch.from_numpy(P.drop_keep(seed, salt, p, np.arange(n))).cuda()


def _next_salt(s):
    """attention_launch.next_salt's recurrence"""
    return (s * 1103515245 + 12345) & 0x7FFFFFFF


# ================================================================== LayerNorm
LN_NV = tuple(range(1, 9))
# 5 rows: one partial forward block and one backward block; 165 rows: 21 forward blocks, the last with 5 rows, and
# 3 backward blocks, the last with 37
LN_ROWS = (5, 165)
LN_VARIANTS = ("plain", "pos", "mapped", "join")
LN_CASES = [(v, nv, rows) for v in LN_VARIANTS for nv in LN_NV for rows in LN_ROWS]
LN_HALF_CASES = [(nv, rows) for nv in LN_NV for rows in LN_ROWS]
LN_EMPTY_BWD = LN_NV


def _ln_inputs(rows, c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(rows, c, device="cuda", generator=g) * 3 + 1
    x += torch.randn(rows, 1, device="cuda", generator=g) * 4           # rows with their own offset
    gamma = 1 + 0.2 * torch.randn(c, device="cuda", generator=g)
    beta = 0.2 * torch.randn(c, device="cuda", generator=g)
    return x, gamma, beta, g


def _ln_ref(x, gamma, beta):
    xd = x.double()
    mean = xd.mean(1)
    rstd = 1.0 / torch.sqrt(xd.var(1, unbiased=False) + EPS)
    xh = (xd - mean[:, None]) * rstd[:, None]
    return xh * gamma.double() + beta.double(), mean, rstd, xh


def _ln_bwd_ref(d, xh, rstd, gamma):
    dxh = d * gamma.double()
    c = d.shape[1]
    dx = rstd[:, None] * (dxh - dxh.sum(1, keepdim=True) / c - xh * (dxh * xh).sum(1, keepdim=True) / c)
    return dx, (d * xh).sum(0), d.sum(0)


def _check_stats(tag, mean, rstd, m_ref, r_ref):
    _bar(f"ln {tag} mean", ((mean.double() - m_ref).abs() / (m_ref.abs() + 1)).max(), 1e-6)
    _bar(f"ln {tag} rstd", ((rstd.double() - r_ref).abs() / r_ref).max(), 1e-6)


@pytest.mark.parametrize("variant,nv,rows", LN_CASES)
def test_layer_norm_instances_vs_fp64(variant, nv, rows):
    """forward (y, y + pos, mean, rstd) and backward (dx, dgamma, dbeta) of layer_norm_*_kernel<nv>:
    plain     coda_layer_norm_fwd / coda_layer_norm_bwd
    pos       coda_layer_norm_fwd_ex with y and y + pos
    mapped    y and dy row-mapped ((q, b) -> (b, q) rows of a padded buffer); every other byte must stay as it was
    join      y_pos only (y NULL); backward with dy + dy2 and the by-pass gradient `add`"""
    L = _L()
    c = nv * 128
    x, gamma, beta, g = _ln_inputs(rows, c, 100 * nv + rows)
    y_ref, m_ref, r_ref, xh = _ln_ref(x, gamma, beta)
    mean = torch.full((rows,), float("nan"), device="cuda")
    rstd = torch.full((rows,), float("nan"), device="cuda")
    dy = torch.randn(rows, c, device="cuda", generator=g)
    dy2 = add = None
    d_ref = dy.double()
    if variant == "plain":
        y = torch.empty(rows, c, device="cuda")
        _ok(L.coda_layer_norm_fwd(_ll(rows), _i(c), _f(EPS), _p(x), _p(gamma), _p(beta), _p(y), _p(mean), _p(rstd),
                                  _s()), "layer_norm_fwd")
        _bar("ln y", _rel(y, y_ref), 1e-6)
    elif variant in ("pos", "join"):
        pos = torch.randn(rows, c, device="cuda", generator=g)
        y = torch.empty(rows, c, device="cuda") if variant == "pos" else None
        ypos = torch.empty(rows, c, device="cuda")
        _ok(L.coda_layer_norm_fwd_ex(_ll(rows), _i(c), _f(EPS), _p(x), _p(gamma), _p(beta), _p(y), _i(0), _ll(0),
                                     _ll(0), _p(pos), _p(ypos), _p(mean), _p(rstd), _s()), "layer_norm_fwd_ex")
        if y is not None:
            _bar("ln y", _rel(y, y_ref), 1e-6)
        _bar("ln y+pos", _rel(ypos, y_ref + pos.double()), 1e-6)
    else:
        b = 3 if rows % 3 == 0 else 1
        q = rows // b
        w = c + 64                                   # padded rows, and one spare row per b: (b, q + 1, c + 64)
        so, si = w, (q + 1) * w
        sentinel = torch.randn(b, q + 1, w, device="cuda", generator=g)
        buf = sentinel.clone()
        _ok(L.coda_layer_norm_fwd_ex(_ll(rows), _i(c), _f(EPS), _p(x), _p(gamma), _p(beta), _p(buf), _i(b), _ll(so),
                                     _ll(si), None, None, _p(mean), _p(rstd), _s()), "layer_norm_fwd_ex mapped")
        inside = torch.zeros(b, q + 1, w, dtype=torch.bool, device="cuda")
        inside[:, :q, :c] = True
        assert torch.equal(_bits(buf)[~inside], _bits(sentinel)[~inside]), "bytes outside the mapped rows changed"
        got = buf[:, :q, :c].permute(1, 0, 2).reshape(rows, c)        # row r = qi * b + bi lives at [bi, qi]
        _bar("ln y", _rel(got, y_ref), 1e-6)
        # the gradient arrives in the same layout; what lies outside the mapped rows is never read
        dbuf = torch.full((b, q + 1, w), float("nan"), device="cuda")
        dbuf[:, :q, :c] = dy.view(q, b, c).permute(1, 0, 2)
        dy = dbuf
    _check_stats(variant, mean, rstd, m_ref, r_ref)

    nblk_scratch = int(L.coda_layer_norm_bwd_scratch(_ll(rows), _i(c)))
    assert nblk_scratch == P.ln_bwd_blocks(rows) * 2 * c
    partial = torch.empty(nblk_scratch, device="cuda")
    dx = torch.empty(rows, c, device="cuda")
    dgamma = torch.full((c,), float("nan"), device="cuda")
    dbeta = torch.full((c,), float("nan"), device="cuda")
    if variant == "plain":
        _ok(L.coda_layer_norm_bwd(_ll(rows), _i(c), _p(dy), _p(x), _p(gamma), _p(mean), _p(rstd), _p(dx), _p(dgamma),
                                  _p(dbeta), _p(partial), _s()), "layer_norm_bwd")
    else:
        inner, so_, si_ = (b, so, si) if variant == "mapped" else (0, 0, 0)
        if variant == "join":
            dy2 = torch.randn(rows, c, device="cuda", generator=g)
            add = torch.randn(rows, c, device="cuda", generator=g)
            d_ref = d_ref + dy2.double()
        _ok(L.coda_layer_norm_bwd_ex(_ll(rows), _i(c), _p(dy), _i(inner), _ll(so_), _ll(si_), _p(dy2), _p(add), _p(x),
                                     _p(gamma), _p(mean), _p(rstd), _p(dx), _p(dgamma), _p(dbeta), _p(partial), _s()),
            "layer_norm_bwd_ex")
    dx_ref, dg_ref, db_ref = _ln_bwd_ref(d_ref, xh, r_ref, gamma)
    if add is not None:
        dx_ref = dx_ref + add.double()
    _bar("ln dx", _rel(dx, dx_ref), 1e-6)
    _bar("ln dgamma", _rel(dgamma, dg_ref), 1e-6)
    _bar("ln dbeta", _rel(dbeta, db_ref), 1e-6)


@pytest.mark.parametrize("nv", LN_EMPTY_BWD)
def test_layer_norm_backward_of_no_rows_zeroes_dgamma_dbeta(nv):
    L = _L()
    c = nv * 128
    dgamma = torch.full((c,), 7.0, device="cuda")
    dbeta = torch.full((c,), -7.0, device="cuda")
    _ok(L.coda_layer_norm_bwd_ex(_ll(0), _i(c), None, _i(0), _ll(0), _ll(0), None, None, None, None, None, None, None,
                                 _p(dgamma), _p(dbeta), None, _s()), "layer_norm_bwd_ex rows 0")
    assert torch.equal(dgamma, torch.zeros_like(dgamma)) and torch.equal(dbeta, torch.zeros_like(dbeta))


@pytest.mark.parametrize("nv,rows", LN_HALF_CASES)
def test_layer_norm_half_instances_vs_fp64(nv, rows):
    """fp16 in and out: y must be the fp64 value rounded to half, up to the fp32 statistics' error"""
    L = _L()
    c = nv * 128
    x, gamma, beta, _ = _ln_inputs(rows, c, 7 * nv + rows)
    xh16 = x.half()
    y = torch.empty_like(xh16)
    _ok(L.coda_layer_norm_fwd_half(_ll(rows), _i(c), _f(EPS), _p(xh16), _p(gamma), _p(beta), _p(y), _s()),
        "layer_norm_fwd_half")
    ref, _, _, _ = _ln_ref(xh16.float(), gamma, beta)
    yn = y.float().cpu().numpy()
    half_ulp = 0.5 * np.spacing(np.abs(yn).astype(np.float16)).astype(np.float64)
    excess = np.maximum(np.abs(yn.astype(np.float64) - ref.cpu().numpy()) - half_ulp, 0.0)
    _bar("ln half excess over rounding", (excess / np.abs(ref.cpu().numpy()).max()).max(), 2e-7)


# ================================================================== BatchNorm on rows
def _bn_rows_small(c):
    return 3          # with 2 rows the normalised output is +-1 whatever the input, and dy is exactly 0


def _bn_rows_strided(c):
    return P.BN_MAX_BLOCKS * P.bn_slots(c) + P.bn_slots(c) // 2 + 1


BN_CASES = [(c, rows, relu, PS[k % 4] if drop else 0.0)
            for k, c in enumerate(P.BN_WIDTHS) for rows in (_bn_rows_small(c), _bn_rows_strided(c))
            for relu in (False, True) for drop in (False, True)]


@pytest.mark.parametrize("c,rows,relu,p", BN_CASES)
def test_bn_act_rows_vs_fp64(c, rows, relu, p):
    """ops.bn_act_rows (statistics + bn_act_fwd, bn_act_bwd_reduce + bn_act_bwd) against fp64: output, running
    buffers, dy, dgamma and dbeta, with the column means 10 standard deviations from zero; the forward and backward
    dropout masks against the twin, element by element"""
    from coda_neurips2023_b200 import attention_launch as A
    from coda_neurips2023_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(c * 1000 + rows + int(relu))
    bn = torch.nn.BatchNorm1d(c).cuda().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0.0, 0.3)
        bn.running_mean.normal_(0.0, 1.0)
        bn.running_var.uniform_(0.5, 2.0)
    rm0, rv0 = bn.running_mean.double(), bn.running_var.double()
    # every column's own mean sits 10 of its own standard deviations from zero, even with 2 or 3 rows
    zs = torch.randn(rows, c, device="cuda", generator=g)
    zs = (zs - zs.mean(0)) / zs.std(0, unbiased=False)
    y = zs * 1.7 + 17.0
    seed = (c * 7919 + rows) & 0x7FFFFFFF
    A.seed_counter(y.device).fill_(seed)
    salt = _next_salt(A._CALL_SALT) if p > 0 else 0
    h = y.clone().requires_grad_(True)
    out = ops.bn_act_rows(h, bn, relu, p, True)

    yr = y.double().requires_grad_(True)
    wr = bn.weight.detach().double().requires_grad_(True)
    br = bn.bias.detach().double().requires_grad_(True)
    mean, var = yr.detach().mean(0), yr.detach().var(0, unbiased=False)
    z = (yr - yr.mean(0)) / torch.sqrt(yr.var(0, unbiased=False) + bn.eps) * wr + br
    a = torch.relu(z) if relu else z
    keep = _keep(seed, salt, p, rows * c).view(rows, c)
    mult = keep.double() * float(P.drop_scale(p)) if p > 0 else torch.ones_like(a)
    ref = a * mult
    _bar("bn out", _rel(out, ref.detach()), 1.8e-5)
    _bar("bn running_mean", _rel(bn.running_mean, 0.9 * rm0 + 0.1 * mean), 1e-6)
    _bar("bn running_var", _rel(bn.running_var, 0.9 * rv0 + 0.1 * var * rows / (rows - 1)), 1e-5)
    zd = z.detach()
    clear = zd.abs() > 1e-3 if relu else torch.ones_like(keep)     # where fp32 and fp64 agree on the ReLU
    if p > 0:
        live = clear & (a.detach().abs() > 1e-3)
        assert torch.equal((out != 0)[live], keep[live]), "forward mask differs from the twin"

    gout = torch.randn(rows, c, device="cuda", generator=g)
    gout = torch.where(gout >= 0, 0.5 + gout, gout - 0.5)            # |dout| >= 0.5: the mask reads off dy below
    gout = torch.where(clear, gout, torch.zeros_like(gout))
    out.backward(gout)
    ref.backward(gout.double())
    _bar("bn dy", _rel(h.grad, yr.grad), 2e-5)
    _bar("bn dgamma", _rel(bn.weight.grad, wr.grad), 2e-5)
    _bar("bn dbeta", _rel(bn.bias.grad, br.grad), 1.5e-6)
    if p > 0:
        # dy = k (dz - s1 / n - xhat s2 / n): rebuild dz from the kernel's dy, dgamma and dbeta
        invstd = 1.0 / torch.sqrt(var + bn.eps)
        k = bn.weight.double() * invstd
        xhat = (y.double() - mean) * invstd
        dz = h.grad.double() / k + bn.bias.grad.double() / rows + xhat * bn.weight.grad.double() / rows
        on = clear & (gout != 0) & ((zd > 0) if relu else torch.ones_like(keep))
        got_keep = dz.abs() > 0.5 * gout.double().abs() * float(P.drop_scale(p))
        assert torch.equal(got_keep[on], keep[on]), "backward mask differs from the twin"


# ================================================================== dropout / residual + dropout
_STRIDED_N = 4 * (P.STREAM_CAP * P.THREADS + 1)          # the smallest n whose float4 loop takes a second step
DROP_CASES = [(n, PS[k % 4], seed, salt) for k, (n, seed, salt) in enumerate([
    (4096, 0, 12345), (1025, 7919, 0x7FFFFFFF), (1026, 0xFFFFFFFF, 1), (1027, 2 * 7919, 987654321),
    (_STRIDED_N, 3 * 7919, 5), (_STRIDED_N + 1, 0x80000000, 1103527590), (_STRIDED_N + 2, 123456789, 77),
    (_STRIDED_N + 3, 4 * 7919, 2 ** 31 - 2)])] + [(3, 0.5, 11, 13), (1027, 0.1, 7919 * 5, 12345)]


@pytest.mark.parametrize("n,p,seed,salt", DROP_CASES)
def test_dropout_kernels_mask_equals_twin(n, p, seed, salt):
    """coda_dropout_add_fwd with and without a residual, and coda_dropout_bwd: the keep mask equals the twin's element
    by element; the values equal fp64 within fp32 rounding"""
    L = _L()
    g = torch.Generator(device="cuda").manual_seed(n + seed)
    x = torch.rand(n, device="cuda", generator=g) + 0.5
    x = torch.where(torch.rand(n, device="cuda", generator=g) < 0.5, -x, x)
    r = torch.randn(n, device="cuda", generator=g)
    sd = _seed_tensor(seed)
    keep = _keep(seed, salt, p, n)
    scale = float(P.drop_scale(p))
    for resid in (r, None):
        out = torch.full((n,), float("nan"), device="cuda")
        _ok(L.coda_dropout_add_fwd(_ll(n), _p(x), _p(resid), _f(p), _u(salt), _p(sd), _p(out), _s()), "dropout_add")
        base = resid.double() if resid is not None else torch.zeros(n, dtype=torch.float64, device="cuda")
        got_keep = (out.double() - base).abs() > 0.5 * x.double().abs() * scale
        assert torch.equal(got_keep, keep), f"resid={resid is not None}: mask differs from the twin"
        exp = base + x.double() * keep.double() * scale
        err = ((out.double() - exp).abs() / (base.abs() + x.double().abs() * scale)).max()
        _bar("dropout value", err, 4e-7)
    dx = torch.full((n,), float("nan"), device="cuda")
    _ok(L.coda_dropout_bwd(_ll(n), _p(x), _f(p), _u(salt), _p(sd), _p(dx), _s()), "dropout_bwd")
    assert torch.equal(dx != 0, keep), "backward mask differs from the twin"
    _bar("dropout value", ((dx.double() - x.double() * keep.double() * scale).abs() / (x.double().abs() * scale)).max(),
         4e-7)


def test_ops_dropout_wiring_hands_forward_and_backward_the_same_salt():
    """through ops: the salt is the next value of attention_launch.next_salt's sequence and the seed the device
    counter, before and after advance_seed; the backward regenerates the forward's mask"""
    from coda_neurips2023_b200 import attention_launch as A
    from coda_neurips2023_b200 import ops

    dev = torch.device("cuda", torch.cuda.current_device())     # the counter ops reads: keyed by "cuda:N"
    n = 8 * 256 * 3 + 3
    g = torch.Generator(device="cuda").manual_seed(5)
    masks = []
    for step in range(2):
        if step:
            A.advance_seed(dev)
        seed = int(A.seed_counter(dev).item()) & 0xFFFFFFFF
        for p, with_resid in ((0.1, True), (0.5, False)):
            salt = _next_salt(A._CALL_SALT)
            x = (torch.rand(n, device="cuda", generator=g) + 0.5).requires_grad_(True)
            r = torch.randn(n, device="cuda", generator=g, requires_grad=True)
            out = ops.dropout_add(x, r, p, True) if with_resid else ops.dropout(x, p, True)
            assert A._CALL_SALT == salt
            keep = _keep(seed, salt, p, n)
            masks.append(keep)
            base = r.detach() if with_resid else torch.zeros_like(out)
            assert torch.equal((out.detach() - base).abs() > 0.5 * x.detach() * float(P.drop_scale(p)), keep)
            gout = torch.rand(n, device="cuda", generator=g) + 0.5
            out.backward(gout)
            assert torch.equal(x.grad != 0, keep)
            exp = gout.double() * keep.double() * float(P.drop_scale(p))
            _bar("dropout value", ((x.grad.double() - exp).abs() / exp.abs().clamp_min(1e-30)).max(), 4e-7)
            if with_resid:
                assert torch.equal(r.grad, gout)
    assert not torch.equal(masks[0], masks[2])           # the advanced seed draws a new mask


# ================================================================== clip + AdamW
BETAS, ADAM_EPS, LR = (0.9, 0.999), 1e-8, 3e-3
# the C ABI takes the betas as fp32: the restatement uses the same values (0.999 in fp32 is 0.999 + 1.3e-8, which
# moves 1 - beta2 at step 1 by 1.3e-5 relative)
BETAS32 = tuple(float(np.float32(b)) for b in BETAS)
ADAMW_N = 4 * P.NORM_BLOCKS * P.THREADS + 4099          # grid-strided norm, n % 4 == 3


def _adamw_chunks():
    """(offset, len, weight_decay) of hand-built chunks: every (head, tail) pair around a float4 body, tensors of 1-3
    elements, inactive gaps between chunks, and one tensor split into three chunks"""
    rng = np.random.default_rng(5)
    wds = (0.0, 0.05)
    chunks, off, k = [], 3, 0
    for mis in range(4):
        for tail in range(4):
            off += (mis - off) % 4
            head = (4 - mis) % 4
            ln = head + 4 * int(rng.integers(1, 80)) + tail
            chunks.append((off, ln, wds[k % 2]))
            k += 1
            off += ln + 1 + int(rng.integers(0, 6))
    for ln in (1, 2, 3, 1, 2, 3, 3):
        chunks.append((off, ln, wds[k % 2]))
        k += 1
        off += ln + 1 + int(rng.integers(0, 3))
    off += (1 - off) % 4
    for ln in (16384, 16384, 1001):
        chunks.append((off, ln, 0.05))
        off += ln
    assert off < ADAMW_N
    return chunks


ADAMW_CHUNKS = _adamw_chunks()
ADAMW_RUNS = [(steps, clip, gs, 0) for steps in (1, 20) for clip in ("off", "above", "below") for gs in (1.0, 0.25)]
ADAMW_RUNS += [(3, "below", 0.25, 10 ** 4)]           # bias corrections at a large step count


def _chunk_table(chunks):
    from coda_neurips2023_b200.engine import FlatAdamW

    arr = (FlatAdamW._Chunk * len(chunks))()
    for k, (off, ln, wd) in enumerate(chunks):
        arr[k].offset, arr[k].len, arr[k].weight_decay = off, ln, wd
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).clone().cuda()


@pytest.mark.parametrize("steps,clip,gs,start", ADAMW_RUNS)
def test_clip_adamw_chunks_vs_fp64(steps, clip, gs, start):
    """coda_grad_norm + coda_adamw_update against an fp64 restatement of clip_grad_norm_ + torch.optim.AdamW, over
    hand-built chunk tables; state[0..4] too; every element outside the chunks keeps its bits"""
    L = _L()
    n = ADAMW_N
    g = torch.Generator(device="cuda").manual_seed(steps * 10 + len(clip) + int(gs * 4))
    param = torch.randn(n, device="cuda", generator=g)
    m = torch.randn(n, device="cuda", generator=g) * 1e-3
    v = torch.rand(n, device="cuda", generator=g) * 1e-5
    p0, m0, v0 = param.clone(), m.clone(), v.clone()
    idx = torch.cat([torch.arange(o, o + ln, device="cuda") for o, ln, _ in ADAMW_CHUNKS])
    wd = torch.cat([torch.full((ln,), w, dtype=torch.float64, device="cuda") for _, ln, w in ADAMW_CHUNKS])
    outside = torch.ones(n, dtype=torch.bool, device="cuda")
    outside[idx] = False
    pd, md, vd = param.double()[idx], m.double()[idx], v.double()[idx]
    expected = (n ** 0.5) * 1e-2 * abs(gs)
    max_norm = {"off": 0.0, "above": 2.0 * expected, "below": 0.25 * expected}[clip]
    state = torch.zeros(8, device="cuda")
    state[0] = start
    scratch = torch.empty(int(L.coda_grad_norm_scratch_floats()), device="cuda")
    lr_dev = torch.tensor([LR], device="cuda")
    table = _chunk_table(ADAMW_CHUNKS)
    b1, b2 = BETAS32
    for it in range(steps):
        grad = torch.randn(n, device="cuda", generator=g) * 1e-2
        grad[-3:] = 0.3                      # the scalar tail of the norm carries weight
        _ok(L.coda_grad_norm(_ll(n), _p(grad), _f(gs), _f(max_norm), _f(b1), _f(b2), _p(scratch), _p(state), _s()),
            "grad_norm")
        _ok(L.coda_adamw_update(_i(len(ADAMW_CHUNKS)), _p(table), _p(param), _p(grad), _p(m), _p(v), _p(lr_dev),
                                _f(gs), _f(b1), _f(b2), _f(ADAM_EPS), _p(state), _s()), "adamw_update")
        gd = grad.double() * gs
        norm = gd.norm().item()
        coef = min(max_norm / (norm + 1e-6), 1.0) if max_norm > 0 else 1.0
        t = start + it + 1
        ge = gd[idx] * coef
        pd = pd * (1.0 - LR * wd)
        md = b1 * md + (1 - b1) * ge
        vd = b2 * vd + (1 - b2) * ge * ge
        bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
        pd = pd - (LR / bc1) * md / (vd.sqrt() / bc2 ** 0.5 + ADAM_EPS)
        st = state.double().cpu()
        assert st[0].item() == t
        _bar("adamw norm", abs(st[1].item() - norm) / norm, 1e-6)
        _bar("adamw coef", abs(st[2].item() - coef) / coef, 1e-6)
        _bar("adamw bias corrections", max(abs(st[3].item() - bc1) / bc1, abs(st[4].item() - bc2 ** 0.5) / bc2 ** 0.5),
             2e-7)
        if clip == "below":
            assert coef < 0.5
        elif clip == "above":
            assert coef == 1.0
    _bar("adamw param / lr", (param.double()[idx] - pd).abs().max().item() / LR, 4e-3)
    _bar("adamw exp_avg", _rel(m[idx], md), 1e-6)
    _bar("adamw exp_avg_sq", _rel(v[idx], vd), 1.5e-6)
    for got, before in ((param, p0), (m, m0), (v, v0)):
        assert torch.equal(_bits(got)[outside], _bits(before)[outside]), "an element outside the chunks changed"


NORM_NS = (1, 2, 3, 4, 7, 1029, 4 * P.NORM_BLOCKS * P.THREADS + 4, 4 * P.NORM_BLOCKS * P.THREADS * 2 + 1,
           4 * P.NORM_BLOCKS * P.THREADS * 2 + 2, 4 * P.NORM_BLOCKS * P.THREADS * 2 + 3)


@pytest.mark.parametrize("n", NORM_NS)
def test_grad_norm_tail_and_grid_stride_vs_fp64(n):
    """state[1] = |grad_scale| * ||grad||, the clip coefficient and the step counter; the scalar tail elements are the
    largest of the buffer, so leaving them out moves the norm far past the bar"""
    L = _L()
    g = torch.Generator(device="cuda").manual_seed(n)
    grad = torch.randn(n, device="cuda", generator=g) * 1e-2
    if n & 3:
        grad[-(n & 3):] = 2.0
    state = torch.zeros(8, device="cuda")
    scratch = torch.empty(int(L.coda_grad_norm_scratch_floats()), device="cuda")
    gs, max_norm = -0.5, 0.5
    _ok(L.coda_grad_norm(_ll(n), _p(grad), _f(gs), _f(max_norm), _f(0.9), _f(0.999), _p(scratch), _p(state), _s()),
        "grad_norm")
    norm = grad.double().norm().item() * abs(gs)
    st = state.double().cpu()
    assert st[0].item() == 1.0
    _bar("adamw norm", abs(st[1].item() - norm) / norm, 1e-6)
    coef = min(max_norm / (norm + 1e-6), 1.0)
    _bar("adamw coef", abs(st[2].item() - coef) / coef, 1e-6)


# ================================================================== Hungarian
def _step_nactual():
    from coda_neurips2023_b200 import synthetic

    batch = synthetic.make_batch(8, 2048, seed=3)
    return np.tile(batch["gt_box_present"].sum(1).astype(np.int32), 7)     # 7 auxiliary layers, layer-major


# (nprop, ngt, nactual per scene, integer costs)
HUNG_CASES = [
    (1024, 64, [64, 30, 73, 0, 1], False),               # unstaged, gt x proposals; 73 > ngt
    (64, 1024, [1024, 64, 100, 30, 1100, 0], False),      # unstaged, proposals x gt (na >= nprop) and transposed (30)
    (1024, 64, [64, 17, 64], True),                       # unstaged ties
    (64, 1024, [1024, 64, 30], True),
    (256, 64, [64, 20, 70, 0], False),                    # staged, transposed
    (16, 64, [64, 16, 5, 70], False),                     # staged, proposals x gt and transposed
    (16, 64, [64, 16, 5], True),
    (256, 64, "step", False),                             # the step's auxiliary call: 7 layers x 8 scenes
]


@pytest.mark.parametrize("case", range(len(HUNG_CASES)))
def test_hungarian_paths_equal_scipy(case):
    from scipy.optimize import linear_sum_assignment

    from coda_neurips2023_b200 import ops

    nprop, ngt, nact, ints = HUNG_CASES[case]
    nact = _step_nactual() if isinstance(nact, str) else np.array(nact, np.int32)
    b = len(nact)
    rng = np.random.default_rng(case)
    if ints:
        cost = rng.integers(0, 4, size=(b, nprop, ngt)).astype(np.float32)
    else:
        cost = rng.standard_normal((b, nprop, ngt)).astype(np.float32)
    inds, mask = ops.hungarian(torch.from_numpy(cost).cuda(), torch.from_numpy(nact).cuda())
    inds, mask = inds.cpu().numpy(), mask.cpu().numpy()
    for i in range(b):
        na = min(int(nact[i]), ngt)
        e_inds = np.zeros(nprop, np.int64)
        e_mask = np.zeros(nprop, np.float32)
        if na > 0:
            r, c = linear_sum_assignment(cost[i, :, :na])
            e_inds[r] = c
            e_mask[r] = 1
        assert np.array_equal(mask[i], e_mask), f"scene {i}: matched set differs"
        assert np.array_equal(inds[i], e_inds), f"scene {i}: assignment differs"


# ================================================================== remainders
SOFTMAX_CASES = [(13, 1), (13, 31), (21, 32), (13, 33), (13, 1025), (5, 3000), (8, 1)]


@pytest.mark.parametrize("rows,c", SOFTMAX_CASES)
def test_softmax_rows_widths_vs_fp64(rows, c):
    from coda_neurips2023_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(rows * c)
    x = torch.randn(rows, c, device="cuda", generator=g) * 5
    x[:, 0] += 30.0                                                     # a dominant first column
    xd = x.double()
    _bar("softmax", (ops.softmax_rows(x).double() - torch.softmax(xd, -1)).abs().max(), 1e-6)
    ref = torch.log_softmax(xd, -1)
    _bar("log_softmax", ((ops.softmax_rows(x, log=True).double() - ref).abs() / (1 + ref.abs())).max(), 1e-6)


# (n, operands, index of the operand `out` aliases or None)
SUM_CASES = [(1027, 17, None), (1027, 17, 0), (1027, 17, 16), (4098, 33, 5), (4098, 33, 32), (4099, 33, 20)]


@pytest.mark.parametrize("n,count,alias", SUM_CASES)
def test_sum_tensors_many_operands_vs_fp64(n, count, alias):
    from coda_neurips2023_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(n + count)
    ts = [torch.randn(n, device="cuda", generator=g) for _ in range(count)]
    ref = torch.stack([t.double() for t in ts]).sum(0)
    out = None if alias is None else ts[alias]
    got = ops.sum_tensors(ts, out=out)
    if out is not None:
        assert got.data_ptr() == out.data_ptr()
    _bar("sum_tensors", _rel(got, ref), 1e-6)


@pytest.mark.parametrize("nl,b,q,d", [(3, 2, 37, 64), (2, 1, 5, 4), (2, 0, 5, 64), (1, 3, 0, 8)])
def test_masked_l1_fractional_weights_and_no_rows_vs_fp64(nl, b, q, d):
    from coda_neurips2023_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(nl * 100 + q)
    pred = torch.randn(nl, b, q, d, device="cuda", generator=g).requires_grad_(True)
    target = torch.randn(b, q, d, device="cuda", generator=g)
    w = torch.rand(b, q, 1, device="cuda", generator=g)
    out = ops.masked_l1(pred, target, w)
    pr = pred.detach().double().requires_grad_(True)
    ref = (pr * w.double() - target.double() * w.double()).abs().sum(dim=(1, 2, 3))
    gl = torch.rand(nl, device="cuda", generator=g) + 0.5
    (got,) = torch.autograd.grad(out, pred, gl)
    if b * q == 0:
        assert torch.equal(out, torch.zeros(nl, device="cuda")) and got.shape == pred.shape
        return
    _bar("masked_l1", ((out.double() - ref).abs() / ref).max(), 1e-6)
    (exp,) = torch.autograd.grad(ref, pr, gl.double())
    _bar("masked_l1 grad", _rel(got, exp), 2e-7)
