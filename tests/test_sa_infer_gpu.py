"""GPU checks of the inference kernel for the pre-encoder's shared MLP + max over neighbours (csrc/sa_infer_sm90.cu,
sa_mlp.shared_mlp_max_infer): against the module-by-module definition (Conv2d 1x1 -> eval-mode BatchNorm2d -> ReLU,
F.max_pool2d over nsample) run in fp64 by PyTorch, at edge shapes and at the evaluation shape (48 scenes x 2048
seeds x 64 neighbours); determinism, memory, and which calls the kernel declines."""
import copy

import pytest
import torch
import torch.nn.functional as F

from coda_neurips2023_b200 import ops, sa_mlp
from coda_neurips2023_b200.pointnet2 import pointnet2_modules as pm
from coda_neurips2023_b200.pointnet2 import pytorch_utils as pt_utils

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _eval_mlp(c0, seed):
    """The pre-encoder's MLP in eval mode with non-trivial running statistics and some negative gamma."""
    torch.manual_seed(seed)
    mlp = pt_utils.SharedMLP([c0, 64, 128, 256], bn=True).cuda().eval()
    for m in mlp.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(-1.5, 1.5)
            m.bias.data.uniform_(-0.3, 0.3)
            m.running_mean.uniform_(-0.5, 0.5)
            m.running_var.uniform_(0.3, 3.0)
    assert any((m.weight < 0).any() for m in mlp.modules() if isinstance(m, torch.nn.BatchNorm2d))
    return mlp


def _reference(mlp, x):
    """fp64 module path: (B, C0, npoint, nsample) -> (B, 256, npoint)"""
    ref = copy.deepcopy(mlp).double()
    with torch.no_grad():
        feats = torch.nn.Sequential.forward(ref, x.double())
        return F.max_pool2d(feats, kernel_size=[1, feats.size(3)]).squeeze(-1)


@pytest.mark.parametrize("c0", [3, 6])
@pytest.mark.parametrize("b,npoint,strided", [
    (1, 1, False),         # one seed: one warpgroup of one CTA has work
    (2, 37, True),         # odd seed count (tail warpgroup), channel slice of a wider tensor (non-packed strides)
    (3, 2048, False),      # many seeds per warpgroup
])
def test_infer_kernel_matches_fp64_modules(c0, b, npoint, strided):
    mlp = _eval_mlp(c0, seed=c0 * 1000 + npoint)
    if strided:
        x = torch.randn(b, c0 + 2, npoint, 64, device="cuda")[:, 1:1 + c0]
        assert not x.is_contiguous()
    else:
        x = torch.randn(b, c0, npoint, 64, device="cuda")
    with torch.no_grad():
        out = mlp.forward_max_pooled_infer(x)
    assert out is not None, "the inference kernel must apply to this layout"
    exp = _reference(mlp, x)
    assert out.shape == exp.shape == (b, 256, npoint)
    scale = exp.abs().max().item()
    err = (out.double() - exp).abs().max().item()
    print(f"PARITY sa_infer c0={c0} seeds={b * npoint}: max err {err / scale:.2e} of max|expected| (bar 1e-4)")
    assert err < 1e-4 * scale


def test_infer_kernel_at_eval_shape():
    """48 scenes x 2048 seeds x 64 neighbours: 512 sampled seeds against an fp64 restatement of those seeds, two runs
    bit-identical, and no memory beyond the pooled output and the weight planes."""
    mlp = _eval_mlp(3, seed=48)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand((48, 3, 2048, 64), device="cuda", generator=g) * 2 - 1      # normalised ball coordinates
    ops.invalidate_weight_cache()          # the measured call packs the weight planes itself
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        out = mlp.forward_max_pooled_infer(x)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert out is not None
    planes = sum(ops._packed_weight(blk.conv.weight.reshape(blk.conv.weight.shape[0], -1), False,
                                    ops.DEFAULT_NSPLIT).nbytes for blk in list(mlp)[1:])
    bar = out.numel() * 4 + planes + (1 << 20)
    print(f"sa_infer peak memory increase {peak / 2**20:.1f} MiB (bar {bar / 2**20:.1f} MiB)")
    assert peak <= bar

    with torch.no_grad():
        again = mlp.forward_max_pooled_infer(x)
    assert torch.equal(out, again), "two runs must give the same bits"

    sel = torch.randperm(48 * 2048, generator=torch.Generator().manual_seed(1))[:512].cuda()
    bs, ps = sel // 2048, sel % 2048
    xs = x[bs, :, ps, :].permute(1, 0, 2).unsqueeze(0)                        # (1, 3, 512, 64)
    exp = _reference(mlp, xs)[0].t()                                           # (512, 256)
    got = out[bs, :, ps]
    scale = exp.abs().max().item()
    err = (got.double() - exp).abs().max().item()
    print(f"PARITY sa_infer eval shape (512 sampled seeds): max err {err / scale:.2e} of max|expected| (bar 1e-4)")
    assert err < 1e-4 * scale


def test_infer_kernel_follows_changed_running_statistics():
    """The folded BatchNorm affine is taken from the module every call: a changed statistic is never stale."""
    mlp = _eval_mlp(3, seed=5)
    x = torch.randn(2, 3, 64, 64, device="cuda")
    with torch.no_grad():
        first = mlp.forward_max_pooled_infer(x)
        mlp[2].bn.bn.running_mean.add_(0.25)
        mlp[1].bn.bn.running_var.mul_(2.0)
        second = mlp.forward_max_pooled_infer(x)
    exp = _reference(mlp, x)
    assert not torch.equal(first, second)
    assert (second.double() - exp).abs().max().item() < 1e-4 * exp.abs().max().item()


def _declined_cases():
    """(name, mlp, x, grad_enabled) the inference kernel must decline"""
    x = torch.randn(2, 3, 16, 64, device="cuda")
    train = _eval_mlp(3, seed=1).train()
    trainable = _eval_mlp(3, seed=2)                                  # eval-mode BN, parameters require grad
    interim = pt_utils.SharedMLP([259, 256, 256, 256], bn=True).cuda().eval()     # masked encoder's interim SA
    no_grad_params = _eval_mlp(3, seed=3)
    for p in no_grad_params.parameters():
        p.requires_grad_(False)
    return [
        ("train-mode BatchNorm under no_grad", train, x, False),
        ("eval-mode BatchNorm, trainable parameters, grad enabled", trainable, x, True),
        ("interim SA of the masked encoder", interim, torch.randn(2, 259, 16, 32, device="cuda"), False),
        ("input requires grad", no_grad_params, x.clone().requires_grad_(True), True),
        ("group of 32", _eval_mlp(3, seed=4), torch.randn(2, 3, 16, 32, device="cuda"), False),
        ("four input channels", _eval_mlp(4, seed=6), torch.randn(2, 4, 16, 64, device="cuda"), False),
        ("other widths", pt_utils.SharedMLP([3, 64, 256, 256], bn=True).cuda().eval(), x, False),
        ("no BatchNorm (conv bias)", pt_utils.SharedMLP([3, 64, 128, 256], bn=False).cuda().eval(), x, False),
        ("CPU input", _eval_mlp(3, seed=8).cpu(), x.cpu(), False),
    ]


@pytest.mark.parametrize("idx", range(9))
def test_infer_path_declines_what_it_does_not_cover(idx):
    name, mlp, x, grad = _declined_cases()[idx]
    with torch.set_grad_enabled(grad):
        assert mlp.forward_max_pooled_infer(x) is None, name


def _sa_module(use_color=False):
    torch.manual_seed(11)
    sa = pm.PointnetSAModuleVotes(radius=0.2, nsample=64, npoint=512, mlp=[3 * int(use_color), 64, 128, 256],
                                  normalize_xyz=True).cuda()
    for m in sa.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(-1.5, 1.5)
            m.bias.data.uniform_(-0.3, 0.3)
            m.running_mean.uniform_(-0.5, 0.5)
            m.running_var.uniform_(0.3, 3.0)
    return sa


def _module_path(sa, xyz, features):
    """PointnetSAModuleVotes.forward written out with the module-by-module MLP (no fused node)"""
    inds = pm.pointnet2_utils.furthest_point_sample(xyz, sa.npoint)
    new_xyz = pm.pointnet2_utils.gather_operation(xyz.transpose(1, 2).contiguous(), inds).transpose(1, 2).contiguous()
    grouped, _ = sa.grouper(xyz, new_xyz, features)
    feats = sa.mlp_module(grouped)
    return F.max_pool2d(feats, kernel_size=[1, feats.size(3)]).squeeze(-1)


@pytest.mark.parametrize("mode", ["train_no_grad", "eval_trainable"])
def test_declined_calls_through_the_sa_module_are_the_module_path_bits(mode, monkeypatch):
    sa = _sa_module()
    xyz = torch.rand(2, 4000, 3, device="cuda")
    calls = []
    monkeypatch.setattr(sa_mlp, "shared_mlp_max_infer", lambda *a: calls.append(1))
    if mode == "train_no_grad":
        sa.train()
        twin = copy.deepcopy(sa)
        with torch.no_grad():
            _, got, _ = sa(xyz)
            exp = _module_path(twin, xyz, None)
    else:
        sa.eval()
        twin = copy.deepcopy(sa)
        _, got, _ = sa(xyz)
        exp = _module_path(twin, xyz, None)
    assert not calls
    assert torch.equal(got, exp)


@pytest.mark.parametrize("use_color", [False, True])
def test_eval_sa_module_takes_the_kernel_and_matches_the_module_path(use_color, monkeypatch):
    sa = _sa_module(use_color).eval()
    xyz = torch.rand(2, 4000, 3, device="cuda")
    features = torch.rand(2, 3, 4000, device="cuda") if use_color else None
    calls = []
    real = sa_mlp.shared_mlp_max_infer
    monkeypatch.setattr(sa_mlp, "shared_mlp_max_infer", lambda *a: calls.append(1) or real(*a))
    with torch.no_grad():
        _, got, _ = sa(xyz, features)
        assert len(calls) == 1
        exp = _module_path(sa, xyz, features)
    assert got.shape == exp.shape == (2, 256, 512)
    assert (got - exp).abs().max().item() < 1e-4 * exp.abs().max().item()
