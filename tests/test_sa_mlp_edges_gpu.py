"""The fused shared-MLP + max-pool node (sa_mlp._SharedMLPMax) and the row kernels of csrc/sa_mlp_kernels.cu against
float64, at the training step's shape, every small-K instance, every channel width, every backward branch, grid-strided
loops and exact ties in the max-pool.

The node's fp64 reference is routed by the kernel's arg-max: the fp64 features are gathered at the rows the kernel
chose, not max-pooled again.  With thousands of groups, a few near-ties within fp32 error are expected, and each would
move a whole pooled gradient entry to another row.  Wherever the kernel's arg-max is not the fp64 first arg-max, the
two fp64 values must agree to the forward bar; exact duplicate rows must resolve to the lowest index.

tests/test_sa_mlp_paths_cpu.py checks, without a GPU, that the case lists below reach every kernel instance, width,
backward branch and grid-strided loop (rules restated in tests/sa_mlp_paths.py).

Every bar is at least 3x the worst error measured over its case list on an H100 80GB HBM3 (400 W power limit); the
measured worst is noted beside each bar."""
import copy
import ctypes

import pytest
import torch

import sa_mlp_paths as P

pytestmark = pytest.mark.gpu

_i, _ll, _f = ctypes.c_int, ctypes.c_longlong, ctypes.c_float


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _ok(err, bar, what):
    assert err < bar, f"{what}: {err:.3e} >= {bar:.1e}"


def _rel(got, exp):
    return float((got.double() - exp).abs().max() / exp.abs().max().clamp_min(1e-30))


def _sum_rel(got, terms):
    """error of column sums over rows, on the scale of the summed magnitudes (sums of random signs cancel)"""
    return float(((got.double() - terms.sum(0)).abs() / terms.abs().sum(0).clamp_min(1e-30)).max())


# ====================================================================== the node

# (spec, b, npoint, group, x_grad, ties): groups = b * npoint rows of `group` neighbours each
NODE_CASES = [
    ([3, 64, 128, 256], 3, 1365, 64, False, False),   # the step's pre-encoder: 4095 groups (> 1056), last 128-row
                                                      # GEMM tile half full
    ([3, 64, 128, 256], 2, 300, 64, False, True),     # ... with ball-query padding: later rows copy the first
    ([6, 64, 128, 256], 2, 517, 64, False, False),    # use_color: 3 xyz + 3 colour channels
    ([1, 512], 3, 41, 16, False, False),              # single small-K block, 2 row slots, pooled gradient expanded
    ([2, 64, 128], 1, 41, 128, False, False),         # POOLED_PRE, group 128
    ([4, 64, 4], 2, 77, 16, False, False),            # last layer 4: the dX GEMM contracts k = 4
    ([5, 64, 256], 1, 37, 256, False, False),         # POOLED_PRE, group 256
    ([7, 64, 128, 256], 1, 101, 96, False, False),    # group 96 tiles 32 but not 128: expand
    ([8, 1024], 2, 53, 7, False, False),              # single small-K block, 1 row slot, odd group
    ([64, 128], 1, 45, 7, True, False),               # GEMM first layer, expand at group 7, input gradient
    ([64, 128, 256], 1, 333, 32, True, False),        # POOLED_PRE, group 32, input gradient
    ([64, 64, 32], 1, 99, 64, True, False),           # last layer 32 through the GEMMs: expand
]

TIE_COPIES = (1, 2, 3, 4, 17)      # copies of row 0: other row slots, and row 0's own slot at 256 channels


def _mlp(spec, seed):
    from coda_neurips2023_b200.pointnet2 import pytorch_utils as pt_utils

    torch.manual_seed(seed)
    mlp = pt_utils.SharedMLP(list(spec), bn=True).cuda().train()
    for m in mlp.modules():                                             # non-trivial affine / running stats
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.uniform_(-0.3, 0.3)
            m.running_mean.uniform_(-0.1, 0.1)
            m.running_var.uniform_(0.8, 1.2)
    return mlp


def _blocks(mlp):
    """(conv, bn) pairs, as SharedMLP.forward_max_pooled collects them"""
    out = []
    for block in mlp:
        mods = list(block.children())
        out.append((mods[0], mods[1][0]))
    return out


def _node(mlp, x, group):
    from coda_neurips2023_b200 import ops, sa_mlp

    blocks = _blocks(mlp)
    assert sa_mlp.applicable(x, blocks, group)
    params = []
    for conv, bn in blocks:
        params += [conv.weight.reshape(conv.weight.shape[0], -1), bn.weight, bn.bias]
    return sa_mlp._SharedMLPMax.apply(x, group, ops.DEFAULT_NSPLIT, [bn for _, bn in blocks], *params)


def _features64(ref, x64):
    """relu(bn(conv(.))) blocks of an fp64 SharedMLP on channels-last rows; BatchNorm2d over (rows, c, 1, 1) is the
    same batch statistics and running-buffer update as over (B, c, npoint, nsample)"""
    h = x64
    for conv, bn in _blocks(ref):
        c = conv.weight.shape[0]
        h = bn((h @ conv.weight.reshape(c, -1).t()).reshape(-1, c, 1, 1)).reshape(-1, c).relu()
    return h


# Bars at >= 3x the worst measured on an H100 80GB HBM3 over NODE_CASES, the weight-update, GradSink and module tests
NODE_FWD_BAR = 3e-6       # pooled output, on the scale of its largest value (measured 9.0e-7)
NODE_GRAD_BAR = 2.5e-4    # every gradient, on the scale of its largest entry (measured 4.4e-5)
# With duplicated rows a ReLU edge that fp32 and fp64 see on different sides flips once per copy: the layer-0 beta
# gradient of the tie case measured 6.0e-4
NODE_TIE_GRAD_BAR = 2e-3
NODE_BUF_BAR = 1.5e-6     # running_mean / running_var, on the scale of their largest entry (measured 4.5e-7)


def _check_node(mlp, ref, x, group, x_grad, argmax, pooled, gout, copies=None, grad_bar=NODE_GRAD_BAR):
    """compare one node call (already run forward) and its backward against the fp64 twin `ref`"""
    groups = x.shape[0] // group
    x64 = x.detach().double().requires_grad_(x_grad)
    feats = _features64(ref, x64).view(groups, group, -1)
    idx = argmax.long()
    exp = feats.gather(1, idx.unsqueeze(1)).squeeze(1)
    scale = float(exp.detach().abs().max())
    _ok(float((pooled.double() - exp).abs().max()) / scale, NODE_FWD_BAR, "pooled")
    # the kernel's arg-max may differ from the fp64 first arg-max only on a near-tie
    with torch.no_grad():
        first = feats.argmax(1)
        moved = idx != first
        if moved.any():
            vf = feats.gather(1, first.unsqueeze(1)).squeeze(1)
            _ok(float((exp - vf)[moved].abs().max()) / scale, NODE_FWD_BAR, "arg-max off a near-tie")
    if copies is not None:
        assert not torch.isin(idx, torch.tensor(copies, device=idx.device)).any(), "a tie resolved to a later row"

    pooled.backward(gout)
    (exp * gout.double()).sum().backward()
    for (name, p), (_, q) in zip(mlp.named_parameters(), ref.named_parameters()):
        _ok(_rel(p.grad, q.grad), grad_bar, f"grad {name}")
    if x_grad:
        _ok(_rel(x.grad, x64.grad), grad_bar, "input grad")
    for (name, bu), (_, bv) in zip(mlp.named_buffers(), ref.named_buffers()):
        if bu.dtype.is_floating_point:
            _ok(_rel(bu, bv), NODE_BUF_BAR, name)
        else:
            assert torch.equal(bu, bv), name                            # num_batches_tracked


@pytest.mark.parametrize("spec,b,npoint,group,x_grad,ties", NODE_CASES)
def test_node_vs_fp64_routed_by_the_kernels_argmax(spec, b, npoint, group, x_grad, ties):
    mlp = _mlp(spec, sum(spec) + npoint + group)
    ref = copy.deepcopy(mlp).double()
    x = torch.randn(b * npoint * group, spec[0], device="cuda")
    copies = None
    if ties:
        xv = x.view(b * npoint, group, spec[0])
        xv[:, list(TIE_COPIES)] = xv[:, :1]
        copies = list(TIE_COPIES)
    x.requires_grad_(x_grad)
    pooled, argmax = _node(mlp, x, group)
    assert pooled.shape == (b * npoint, spec[-1]) and argmax.dtype == torch.uint8
    gout = torch.randn_like(pooled)
    _check_node(mlp, ref, x, group, x_grad, argmax, pooled, gout, copies,
                NODE_TIE_GRAD_BAR if ties else NODE_GRAD_BAR)
    if ties:
        # the copies do hold the maximum of many (group, channel) pairs: the tie rule was exercised
        assert int((argmax == 0).sum()) > 0.005 * argmax.numel()


def test_node_after_an_in_place_weight_update():
    """The packed weight planes are cached under (data_ptr, _version): an optimiser-style in-place update between two
    calls must reach the second call."""
    spec, group = [3, 64, 128, 256], 64
    mlp = _mlp(spec, 11)
    x = torch.randn(2 * 200 * group, 3, device="cuda")
    pooled, _ = _node(mlp, x, group)
    pooled.backward(torch.randn_like(pooled))
    with torch.no_grad():
        for p in mlp.parameters():
            p.add_(torch.sign(p.grad), alpha=-0.05)                     # Adam's first step: lr * sign(grad)
            p.grad = None
    ref = copy.deepcopy(mlp).double()
    x2 = torch.randn_like(x)
    pooled2, argmax2 = _node(mlp, x2, group)
    _check_node(mlp, ref, x2, group, False, argmax2, pooled2, torch.randn_like(pooled2))


@pytest.mark.parametrize("spec,group,x_grad", [([3, 64, 128, 256], 64, False), ([64, 128, 256], 32, True)])
def test_grad_sink_receives_the_nodes_parameter_gradients(spec, group, x_grad):
    """With an armed ops.GradSink (engine.TrainStep.prepare), dW / dgamma / dbeta land in the flat gradient buffer
    with the bits of the unarmed run, and autograd receives None for them."""
    from coda_neurips2023_b200 import engine, ops

    mlp = _mlp(spec, 5)
    twin = copy.deepcopy(mlp)
    x = torch.randn(2 * 150 * group, spec[0], device="cuda")
    gout = torch.randn(2 * 150, spec[-1], device="cuda")
    xt = x.clone().requires_grad_(x_grad)
    pooled, _ = _node(twin, xt, group)
    pooled.backward(gout)
    expected = [p.grad.clone() for p in twin.parameters()]

    params = list(mlp.parameters())
    sink = ops.GradSink()
    sink.watch(params)
    ops.set_grad_sink(sink)
    try:
        state = copy.deepcopy(mlp.state_dict())
        probe, _ = _node(mlp, x.clone().requires_grad_(x_grad), group)      # count mode: nothing is redirected
        probe.backward(gout)
        mlp.load_state_dict(state)
        for p in params:
            p.grad = None
        flat = engine.FlatParameters(mlp)
        sink.arm(flat.flat_param, flat.flat_grad, [off * 4 for off in flat.offsets])
        ops.invalidate_weight_cache()
        flat.flat_grad.fill_(float("nan"))
        xs = x.clone().requires_grad_(x_grad)
        pooled, _ = _node(mlp, xs, group)
        got = torch.autograd.grad(pooled, params + ([xs] if x_grad else []), gout, allow_unused=True)
    finally:
        ops.set_grad_sink(None)
    assert all(g is None for g in got[:len(params)]), "the node returned a sunk gradient to autograd"
    for p, e, off in zip(params, expected, flat.offsets):
        assert torch.equal(flat.flat_grad[off:off + p.numel()].view_as(p), e)
    if x_grad:
        assert torch.equal(got[-1], xt.grad)


def test_preencoder_module_on_a_padded_scene_vs_fp64(monkeypatch):
    """PointnetSAModuleVotes with the pre-encoder's arguments on a sparse scene, where ball query pads most balls by
    repeating their first neighbour, against an fp64 SharedMLP on the module's own grouped features (an exact
    gather)."""
    from coda_neurips2023_b200 import sa_mlp, synthetic
    from coda_neurips2023_b200.pointnet2 import pointnet2_utils
    from coda_neurips2023_b200.pointnet2.pointnet2_modules import PointnetSAModuleVotes

    torch.manual_seed(3)
    npoint, nsample = 256, 64
    mod = PointnetSAModuleVotes(radius=0.2, nsample=nsample, npoint=npoint, mlp=[0, 64, 128, 256],
                                normalize_xyz=True).cuda().train()
    seeded = _mlp([3, 64, 128, 256], 3)
    mod.mlp_module.load_state_dict(seeded.state_dict())
    ref = copy.deepcopy(mod.mlp_module).double()
    xyz = torch.from_numpy(synthetic.point_clouds(2, 2048, seed=11)).cuda()
    inds = pointnet2_utils.furthest_point_sample(xyz, npoint)
    new_xyz = pointnet2_utils.gather_operation(xyz.transpose(1, 2).contiguous(), inds).transpose(1, 2).contiguous()
    grouped, _ = mod.grouper(xyz, new_xyz, None)                        # (B, 3, npoint, nsample)
    rows = grouped.permute(0, 2, 3, 1).reshape(-1, nsample, 3)
    copy_of_first = (rows[:, 1:] == rows[:, :1]).all(-1)                # (groups, nsample - 1)
    assert copy_of_first.float().mean() > 0.5, "the scene must be sparse enough for ball query to pad"

    seen = {}
    apply = sa_mlp._SharedMLPMax.apply

    def spy(*args):
        out = apply(*args)
        seen["argmax"] = out[1]
        return out

    monkeypatch.setattr(sa_mlp._SharedMLPMax, "apply", spy)
    _, feats, _ = mod(xyz, None, inds)                                  # (B, 256, npoint)
    assert "argmax" in seen, "the module did not take the fused path"
    argmax = seen["argmax"]
    pooled = feats.permute(0, 2, 1).reshape(-1, 256)
    # a padded copy of row 0 never wins: row 0 holds the same value with a lower index
    later = torch.cat([torch.zeros_like(copy_of_first[:, :1]), copy_of_first], 1)
    assert not later.gather(1, argmax.long()).any(), "a tie resolved to a padded copy"
    # pooled is a view of the module's output: its backward runs through the module's permute / reshape
    _check_node(mod.mlp_module, ref, rows.reshape(-1, 3), nsample, False, argmax, pooled, torch.randn_like(pooled))


# ====================================================================== the row kernels in isolation

def _row_counts(c):
    """2 rows (unbiased factor 2), a count that is not a multiple of the slot count, and enough rows for every
    block of the 528-block grid to take a second grid-stride step"""
    s = P.slots(c)
    return (2, s * 37 + 1, 2 * P.MAX_BLOCKS * s + 1)


ROW_CASES = [(c, rows) for c in P.WIDTHS for rows in _row_counts(c)]
# (c, groups, group): 2 groups, an odd count, more groups than the 1056-block max-pool grid
MAXPOOL_CASES = [(c, groups, group) for c in P.WIDTHS for groups, group in ((2, 256), (301, 37), (1100, 9))]
OFFSET_RATIOS = (10, 30)
# the GEMM's column-statistics epilogue serves up to 256 columns (wider GEMM layers are declined by sa_mlp.applicable)
FINALIZE_CASES = [(c, rows) for c, rows in ROW_CASES if c <= 256]


def _L():
    from coda_neurips2023_b200._lib import lib

    return lib()


def _call(name, *args):
    from coda_neurips2023_b200._lib import check, stream_of

    check(getattr(_L(), name)(*args, stream_of(torch.empty(0, device="cuda"))), name)


def _p(t):
    from coda_neurips2023_b200._lib import ptr

    return ptr(t)


def _scratch(c):
    L = _L()
    L.coda_bn_rows_scratch_floats.restype = ctypes.c_longlong
    return torch.empty(int(L.coda_bn_rows_scratch_floats(_i(c))), device="cuda")


def _affine(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mean = torch.randn(c, device="cuda", generator=g) * 0.5 + 0.3
    invstd = torch.rand(c, device="cuda", generator=g) + 0.5
    gamma = torch.rand(c, device="cuda", generator=g) + 0.5
    beta = torch.randn(c, device="cuda", generator=g) * 0.3
    return mean, invstd, gamma, beta


def _stats64(y):
    y64 = y.double()
    m = y64.mean(0)
    return m, y64.var(0, unbiased=False)


STATS_BAR = 1e-6          # measured: variance 1.8e-7, running buffers 1.6e-7, mean 6.7e-8, scale / shift 5.7e-8
EPS, MOMENTUM = 1e-5, 0.1


def _check_stats(rows, c, y, mean, invstd, rm0, rv0, rm, rv, gamma=None, beta=None, scale=None, shift=None):
    """mean on the scale of the rows' RMS; the variance on the scale of E[y^2], the size of the two terms
    E[y^2] - E[y]^2 subtracts (rows whose mean is far from zero are test_bn_rows_stats_with_offset_means);
    running buffers relative; scale / shift against the kernel's own mean and invstd"""
    m64, v64 = _stats64(y)
    ms = v64 + m64 * m64
    _ok(float(((mean.double() - m64).abs() / ms.sqrt().clamp_min(1e-30)).max()), STATS_BAR, "mean")
    var = 1.0 / invstd.double() ** 2 - EPS
    _ok(float(((var - v64).abs() / ms.clamp_min(1e-30)).max()), STATS_BAR, "variance")
    if rm is not None:
        _ok(_rel(rm, (1 - MOMENTUM) * rm0.double() + MOMENTUM * m64), STATS_BAR, "running_mean")
        _ok(_rel(rv, (1 - MOMENTUM) * rv0.double() + MOMENTUM * v64 * rows / (rows - 1)), STATS_BAR, "running_var")
    if scale is not None:
        cpad = (c + 63) // 64 * 64
        sc = gamma.double() * invstd.double()
        _ok(_rel(scale[:c], sc), STATS_BAR, "scale")
        # shift = beta - mean * scale cancels: measured on the scale of |beta| + |mean * scale|
        msc = mean.double() * scale[:c].double()
        den = (beta.double().abs() + msc.abs()).max()
        _ok(float((shift[:c].double() - (beta.double() - msc)).abs().max() / den), STATS_BAR, "shift")
        assert torch.equal(scale[c:cpad], torch.zeros(cpad - c, device="cuda"))
        assert torch.equal(shift[c:cpad], torch.zeros(cpad - c, device="cuda"))


def _rows_with_offsets(rows, c, seed):
    torch.manual_seed(seed)
    return torch.randn(rows, c, device="cuda") * (torch.rand(c, device="cuda") + 0.5) + torch.randn(c, device="cuda")


@pytest.mark.parametrize("c,rows", ROW_CASES)
def test_bn_rows_stats_vs_fp64(c, rows):
    """coda_bn_rows_stats with running buffers, coda_bn_rows_stats_affine without them (scale / shift zero-padded to
    a multiple of 64)"""
    y = _rows_with_offsets(rows, c, rows + c)
    rm0, rv0 = torch.randn(c, device="cuda") * 0.1, torch.rand(c, device="cuda") + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_rows_stats", _ll(rows), _i(c), _p(y), _f(EPS), _f(MOMENTUM), _p(rm), _p(rv), _p(mean), _p(invstd),
          _p(_scratch(c)))
    _check_stats(rows, c, y, mean, invstd, rm0, rv0, rm, rv)

    cpad = (c + 63) // 64 * 64
    gamma, beta = torch.rand(c, device="cuda") + 0.5, torch.randn(c, device="cuda") * 0.3
    scale, shift = torch.full((cpad,), float("nan"), device="cuda"), torch.full((cpad,), float("nan"), device="cuda")
    mean2, invstd2 = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_rows_stats_affine", _ll(rows), _i(c), _p(y), _f(EPS), _f(MOMENTUM), _p(None), _p(None), _p(gamma),
          _p(beta), _p(mean2), _p(invstd2), _p(scale), _p(shift), _p(_scratch(c)))
    assert torch.equal(mean2, mean) and torch.equal(invstd2, invstd)
    _check_stats(rows, c, y, mean2, invstd2, None, None, None, None, gamma, beta, scale, shift)


@pytest.mark.parametrize("c,rows", FINALIZE_CASES)
def test_bn_stats_finalize_on_gemm_partials_vs_fp64(c, rows):
    """coda_bn_stats_finalize on the column-statistics partials of the fp32-A GEMM's epilogue"""
    from coda_neurips2023_b200 import ops

    torch.manual_seed(rows * 3 + c)
    a = torch.randn(rows, 64, device="cuda")
    w = torch.randn(c, 64, device="cuda") / 8
    y, part = ops.gemm_a32(a, ops.pack_split(w, c, 64, 64, 1, 3), c, want_stats=True)
    nblocks = part.shape[0]
    rm0, rv0 = torch.randn(c, device="cuda") * 0.1, torch.rand(c, device="cuda") + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    gamma, beta = torch.rand(c, device="cuda") + 0.5, torch.randn(c, device="cuda") * 0.3
    cpad = (c + 63) // 64 * 64
    scale, shift = torch.full((cpad,), float("nan"), device="cuda"), torch.full((cpad,), float("nan"), device="cuda")
    mean, invstd = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_stats_finalize", _i(nblocks), _ll(rows), _i(c), _p(part), _f(EPS), _f(MOMENTUM), _p(rm), _p(rv),
          _p(gamma), _p(beta), _p(mean), _p(invstd), _p(scale), _p(shift))
    _check_stats(rows, c, y, mean, invstd, rm0, rv0, rm, rv, gamma, beta, scale, shift)
    mean2, invstd2 = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_stats_finalize", _i(nblocks), _ll(rows), _i(c), _p(part), _f(EPS), _f(MOMENTUM), _p(None),
          _p(None), _p(None), _p(None), _p(mean2), _p(invstd2), _p(None), _p(None))
    assert torch.equal(mean2, mean) and torch.equal(invstd2, invstd)


# relative invstd error; measured 1.48e-6 at 10 std and 1.50e-5 at 30 std (an emulation of the kernel's accumulation
# order predicts 1.5e-6 and 1e-5)
OFFSET_BAR = {10: 5e-6, 30: 5e-5}


@pytest.mark.parametrize("ratio", OFFSET_RATIOS)
def test_bn_rows_stats_with_offset_means(ratio):
    """1 M rows at 256 channels whose means lie `ratio` standard deviations from zero: E[y^2] - E[y]^2 from fp32
    per-thread sums loses digits as ratio^2 grows"""
    rows, c = 1 << 20, 256
    torch.manual_seed(ratio)
    sigma = torch.rand(c, device="cuda") + 0.5
    sign = torch.where(torch.rand(c, device="cuda") < 0.5, -1.0, 1.0)
    y = torch.randn(rows, c, device="cuda") * sigma + sign * ratio * sigma
    mean, invstd = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_rows_stats", _ll(rows), _i(c), _p(y), _f(EPS), _f(MOMENTUM), _p(None), _p(None), _p(mean),
          _p(invstd), _p(_scratch(c)))
    m64, v64 = _stats64(y)
    del y
    _ok(float(((mean.double() - m64).abs() / (v64 + m64 * m64).sqrt()).max()), STATS_BAR, "mean")
    _ok(_rel(invstd, 1.0 / torch.sqrt(v64 + EPS)), OFFSET_BAR[ratio], f"invstd at {ratio} std")


MAXPOOL_BAR = 5e-7        # measured 1.0e-7


@pytest.mark.parametrize("c,groups,group", MAXPOOL_CASES)
def test_bn_relu_maxpool_rows_vs_fp64(c, groups, group):
    """pooled values and arg-max; exact duplicates of a group's first row in other row slots, and channels that the
    ReLU zeroes on every row (a tie across the whole group), resolve to the first index"""
    torch.manual_seed(groups + c + group)
    y = torch.randn(groups * group, c, device="cuda")
    yv = y.view(groups, group, c)
    copies = [i for i in sorted({1, P.slots(c), P.slots(c) + 1, group - 1}) if 0 < i < group]
    yv[:, copies] = yv[:, :1]
    mean, invstd, gamma, beta = _affine(c, c + group)
    beta[3::4] = -100.0                                                 # every row negative: ReLU ties at 0
    pooled = torch.empty(groups, c, device="cuda")
    argmax = torch.empty(groups, c, dtype=torch.uint8, device="cuda")
    _call("coda_bn_relu_maxpool_rows", _ll(groups), _i(group), _i(c), _p(y), _p(mean), _p(invstd), _p(gamma),
          _p(beta), _p(pooled), _p(argmax))
    z = torch.relu((y.double() - mean.double()) * invstd.double() * gamma.double() + beta.double())
    z = z.view(groups, group, c)
    idx = argmax.long()
    exp = z.gather(1, idx.unsqueeze(1)).squeeze(1)
    scale = float(exp.abs().max())
    _ok(float((pooled.double() - exp).abs().max()) / scale, MAXPOOL_BAR, "pooled")
    first = z.argmax(1)
    moved = idx != first
    if moved.any():
        vf = z.gather(1, first.unsqueeze(1)).squeeze(1)
        _ok(float((exp - vf)[moved].abs().max()) / scale, MAXPOOL_BAR, "arg-max off a near-tie")
    assert not torch.isin(idx, torch.tensor(copies, device="cuda")).any(), "a duplicate row won over the first"
    # the ReLU-zeroed channels: the whole group ties at 0, the first row wins
    assert not idx[:, 3::4].any() and not pooled[:, 3::4].any()


REDUCE_BAR = 5e-7         # column sums on the scale of the summed magnitudes, dprime (measured 1.3e-7)


def _off_relu_edge(y, mean, invstd, gamma, beta):
    """move every y whose BatchNorm output lies within 1e-3 of the ReLU edge 2e-3 further out, so that fp32 and fp64
    agree on the mask"""
    k = invstd.double() * gamma.double()
    z = (y.double() - mean.double()) * k + beta.double()
    near = z.abs() < 1e-3
    y += (near * torch.where(z < 0, -2e-3, 2e-3) / k).float()
    return y


def _masked(y, d, mean, invstd, gamma, beta):
    xh = (y.double() - mean.double()) * invstd.double()
    z = xh * gamma.double() + beta.double()
    return torch.where(z > 0, d.double(), 0.0), xh


@pytest.mark.parametrize("c,rows", ROW_CASES)
def test_bn_relu_bwd_reduce_vs_fp64(c, rows):
    torch.manual_seed(rows + 7 * c)
    y, dz = torch.randn(rows, c, device="cuda"), torch.randn(rows, c, device="cuda")
    mean, invstd, gamma, beta = _affine(c, rows)
    _off_relu_edge(y, mean, invstd, gamma, beta)
    s1, s2 = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_relu_bwd_reduce", _ll(rows), _i(c), _p(y), _p(dz), _p(mean), _p(invstd), _p(gamma), _p(beta),
          _p(s1), _p(s2), _p(_scratch(c)))
    d, xh = _masked(y, dz, mean, invstd, gamma, beta)
    _ok(_sum_rel(s1, d), REDUCE_BAR, "s1")
    _ok(_sum_rel(s2, d * xh), REDUCE_BAR, "s2")


@pytest.mark.parametrize("c,groups", ROW_CASES)
def test_bn_relu_bwd_reduce_pooled_vs_fp64(c, groups):
    """only the arg-max row of a (group, channel) carries a gradient; dprime = gamma * invstd * the masked gradient"""
    group = 5
    torch.manual_seed(groups + 11 * c)
    y = torch.randn(groups * group, c, device="cuda")
    dp = torch.randn(groups, c, device="cuda")
    arg = torch.randint(0, group, (groups, c), dtype=torch.uint8, device="cuda")
    mean, invstd, gamma, beta = _affine(c, groups)
    _off_relu_edge(y.view(-1, c), mean, invstd, gamma, beta)
    s1, s2 = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    dprime = torch.full((groups, c), float("nan"), device="cuda")
    _call("coda_bn_relu_bwd_reduce_pooled", _ll(groups), _i(group), _i(c), _p(y), _p(dp), _p(arg), _p(mean),
          _p(invstd), _p(gamma), _p(beta), _p(s1), _p(s2), _p(_scratch(c)), _p(dprime))
    ysel = y.view(groups, group, c).gather(1, arg.long().unsqueeze(1)).squeeze(1)
    d, xh = _masked(ysel, dp, mean, invstd, gamma, beta)
    assert 0 < int((d == 0).sum()) < d.numel() or groups == 2
    _ok(_sum_rel(s1, d), REDUCE_BAR, "s1")
    _ok(_sum_rel(s2, d * xh), REDUCE_BAR, "s2")
    _ok(_rel(dprime, gamma.double() * invstd.double() * d), REDUCE_BAR, "dprime")
    t1, t2 = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    _call("coda_bn_relu_bwd_reduce_pooled", _ll(groups), _i(group), _i(c), _p(y), _p(dp), _p(arg), _p(mean),
          _p(invstd), _p(gamma), _p(beta), _p(t1), _p(t2), _p(_scratch(c)), _p(None))
    assert torch.equal(t1, s1) and torch.equal(t2, s2)


COEF_BAR = 5e-7           # measured 1.5e-7


@pytest.mark.parametrize("c,rows", ROW_CASES)
def test_bn_bwd_coefs_vs_fp64(c, rows):
    """alpha = -gamma invstd^2 s2 / N, beta = -gamma invstd s1 / N - alpha mean, zero-padded to a multiple of 64"""
    mean, invstd, gamma, _ = _affine(c, rows + c)
    mean += 2.0                                                         # beta's "- alpha * mean" term matters
    s1, s2 = torch.randn(c, device="cuda") * rows, torch.randn(c, device="cuda") * rows
    cpad = (c + 63) // 64 * 64
    alpha, bcoef = torch.full((cpad,), float("nan"), device="cuda"), torch.full((cpad,), float("nan"), device="cuda")
    _call("coda_bn_bwd_coefs", _i(c), _ll(rows), _p(mean), _p(invstd), _p(gamma), _p(s1), _p(s2), _p(alpha), _p(bcoef))
    sc = gamma.double() * invstd.double()
    a64 = -sc * invstd.double() * s2.double() / rows
    b64 = -sc * s1.double() / rows - a64 * mean.double()
    _ok(_rel(alpha[:c], a64), COEF_BAR, "alpha")
    den = ((sc * s1.double() / rows).abs() + (a64 * mean.double()).abs()).max()
    _ok(float((bcoef[:c].double() - b64).abs().max() / den), COEF_BAR, "beta")
    assert torch.equal(alpha[c:], torch.zeros(cpad - c, device="cuda"))
    assert torch.equal(bcoef[c:], torch.zeros(cpad - c, device="cuda"))


SMALL_K_BAR = 1e-6        # measured: linear 2.5e-7, dW 2.2e-7


@pytest.mark.parametrize("c,rows", ROW_CASES)
def test_small_k_linear_and_backward_vs_fp64(c, rows):
    """coda_rows_linear_small_k and coda_bn_relu_bwd_small_k (dW = sum_r dy[r, c] x[r, k]) at every CIN 1..8"""
    L = _L()
    L.coda_bn_rows_small_k_scratch_floats.restype = ctypes.c_longlong
    mean, invstd, gamma, beta = _affine(c, rows + 3 * c)
    for cin in range(1, 9):
        torch.manual_seed(rows + c + cin)
        x = torch.randn(rows, cin, device="cuda")
        w = torch.randn(c, cin, device="cuda")
        y = torch.empty(rows, c, device="cuda")
        _call("coda_rows_linear_small_k", _ll(rows), _i(cin), _i(c), _p(x), _p(w), _p(y))
        terms = x.double().unsqueeze(1) * w.double()                    # (rows, c, cin)
        err = float(((y.double() - terms.sum(-1)).abs() / terms.abs().sum(-1).clamp_min(1e-30)).max())
        _ok(err, SMALL_K_BAR, f"linear cin {cin}")

        dz = torch.randn(rows, c, device="cuda")
        _off_relu_edge(y, mean, invstd, gamma, beta)
        s1, s2 = torch.randn(c, device="cuda") * rows ** 0.5, torch.randn(c, device="cuda") * rows ** 0.5
        sc = torch.empty(int(L.coda_bn_rows_small_k_scratch_floats(_i(cin), _i(c))), device="cuda")
        dw = torch.full((c, cin), float("nan"), device="cuda")
        _call("coda_bn_relu_bwd_small_k", _ll(rows), _i(cin), _i(c), _p(y), _p(dz), _p(mean), _p(invstd), _p(gamma),
              _p(beta), _p(s1), _p(s2), _p(x), _p(dw), _p(sc))
        d, xh = _masked(y, dz, mean, invstd, gamma, beta)
        k, m1, m2 = gamma.double() * invstd.double(), s1.double() / rows, s2.double() / rows
        dy = k * (d - m1 - xh * m2)
        # on the scale of the magnitudes summed, inside dy too: d - s1/N - xhat s2/N cancels at 2 rows
        mag = (k * (d.abs() + m1.abs() + (xh * m2).abs())).unsqueeze(2) * x.double().abs().unsqueeze(1)
        err = (dw.double() - (dy.unsqueeze(2) * x.double().unsqueeze(1)).sum(0)).abs() / mag.sum(0)
        _ok(float(err.max()), SMALL_K_BAR, f"dW cin {cin}")
