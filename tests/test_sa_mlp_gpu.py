"""GPU parity of the fused shared-MLP + max-pool node (include/coda_sa_mlp.h, sa_mlp.py) against the
module-by-module definition (Conv2d 1x1 -> BatchNorm2d -> ReLU blocks, F.max_pool2d over nsample) run in
fp64 by PyTorch: output, running statistics, and every gradient."""
import copy

import pytest
import torch
import torch.nn.functional as F

from coda_neurips2023_b200.pointnet2 import pytorch_utils as pt_utils

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _reference(mlp64, x64):
    feats = torch.nn.Sequential.forward(mlp64, x64)                     # (B, C, npoint, nsample)
    return F.max_pool2d(feats, kernel_size=[1, feats.size(3)]).squeeze(-1)


@pytest.mark.parametrize("spec,b,npoint,nsample,x_grad", [
    ([3, 64, 128, 256], 2, 37, 16, False),      # the CoDA pre-encoder layout (xyz input, tiny-K first layer)
    ([4, 64, 128], 1, 5, 64, False),            # xyz + one feature channel
    ([64, 64, 128], 2, 19, 8, True),            # a deeper SA level: tensor-core first layer, input gradient
    ([3, 128], 3, 11, 7, False),                # single block, odd group size
])
def test_shared_mlp_max_matches_fp64_modules(spec, b, npoint, nsample, x_grad):
    torch.manual_seed(sum(spec) + npoint)
    mlp = pt_utils.SharedMLP(list(spec), bn=True).cuda().train()
    for m in mlp.modules():                                             # non-trivial affine / running stats
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.uniform_(-0.3, 0.3)
            m.running_mean.uniform_(-0.1, 0.1)
            m.running_var.uniform_(0.8, 1.2)
    ref = copy.deepcopy(mlp).double()
    x = torch.randn(b, spec[0], npoint, nsample, device="cuda")
    x64 = x.double().requires_grad_(x_grad)
    x = x.requires_grad_(x_grad)

    out = mlp.forward_max_pooled(x)
    assert out is not None, "fused path must apply to this layout"
    exp = _reference(ref, x64)
    assert out.shape == exp.shape
    scale = exp.abs().max().item()
    assert (out.double() - exp).abs().max().item() < 1e-4 * scale

    g = torch.randn_like(out)
    out.backward(g)
    exp.backward(g.double())
    for (name, p), (_, q) in zip(mlp.named_parameters(), ref.named_parameters()):
        err = (p.grad.double() - q.grad).abs().max().item() / max(q.grad.abs().max().item(), 1e-12)
        assert err < 5e-3, f"{name}: grad rel err {err:.2e}"
    if x_grad:
        err = (x.grad.double() - x64.grad).abs().max().item() / x64.grad.abs().max().item()
        assert err < 5e-3, f"input grad rel err {err:.2e}"
    for (name, bu), (_, bv) in zip(mlp.named_buffers(), ref.named_buffers()):
        if bu.dtype.is_floating_point:
            assert (bu.double() - bv).abs().max().item() < 1e-5, name
        else:
            assert torch.equal(bu, bv), name                          # num_batches_tracked


def test_fused_path_declines_what_it_does_not_cover():
    mlp = pt_utils.SharedMLP([3, 64, 128], bn=True).cuda()
    x = torch.randn(1, 3, 4, 8, device="cuda")
    mlp.eval()
    assert mlp.forward_max_pooled(x) is None                            # eval mode: running statistics
    mlp.train()
    with torch.no_grad():
        assert mlp.forward_max_pooled(x) is None                        # inference
    assert pt_utils.SharedMLP([3, 64, 128], bn=False).cuda().forward_max_pooled(x) is None   # conv bias, no bn
    # the tiny-K first layer produces no input gradient
    assert mlp.forward_max_pooled(x.clone().requires_grad_(True)) is None
    # cin > 8 and not a multiple of 64; a non-last width that is not a multiple of 64; a group of more than 256 rows
    assert pt_utils.SharedMLP([72, 64], bn=True).cuda().forward_max_pooled(torch.randn(1, 72, 4, 8, device="cuda")) \
        is None
    assert pt_utils.SharedMLP([64, 96, 128], bn=True).cuda().forward_max_pooled(
        torch.randn(1, 64, 4, 8, device="cuda")) is None
    assert mlp.forward_max_pooled(torch.randn(1, 3, 2, 257, device="cuda")) is None
    # GEMM layers wider than 256 columns: the GEMM's column statistics would not fit in its shared memory
    assert pt_utils.SharedMLP([64, 512, 1024], bn=True).cuda().forward_max_pooled(
        torch.randn(1, 64, 4, 32, device="cuda")) is None
    assert mlp.forward_max_pooled(torch.randn(1, 3, 2, 256, device="cuda")) is not None
