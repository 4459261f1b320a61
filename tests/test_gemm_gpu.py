"""wgmma GEMM (include/coda_gemm.h) against a float64 matmul of the same operands."""
import pytest
import torch

from coda_neurips2023_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


def _ref(a, b, bias=None, relu=False):
    c = torch.matmul(a.double(), b.double().transpose(-1, -2))
    if bias is not None:
        c = c + bias.double()
    return c.relu() if relu else c


# error of the split: products carry ~8 / 16 / 24 mantissa bits of each operand
TOL = {1: 1.2e-2, 2: 6e-5, 3: 2e-6}


@pytest.mark.parametrize("nsplit", [2, 1, 3])
@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (256, 128, 256), (300, 200, 100), (2048, 768, 256), (77, 13, 3),
                                   (128, 64, 512), (1000, 512, 512)])
def test_gemm_nt_vs_fp64(nsplit, m, n, k):
    torch.manual_seed(m + n + k)
    a = torch.randn(m, k, device="cuda")
    b = torch.randn(n, k, device="cuda")
    bias = torch.randn(n, device="cuda")
    ap = ops.pack_split(a, m, k, k, 1, nsplit)
    bp = ops.pack_split(b, n, k, k, 1, nsplit)
    c = ops.gemm_nt(ap, bp, m, n, bias=bias)[0]
    ref = _ref(a, b, bias)
    scale = (a.double().abs() @ b.double().abs().t()).max()  # sum |a||b|: the natural error scale
    err = ((c.double() - ref).abs().max() / scale).item()
    assert err < TOL[nsplit], f"nsplit={nsplit} m={m} n={n} k={k}: err {err:.2e}"
    c2 = ops.gemm_nt(ap, bp, m, n, bias=None, relu=True)[0]
    ref2 = _ref(a, b, None, True)
    assert ((c2.double() - ref2).abs().max() / scale).item() < TOL[nsplit]


def test_gemm_transposed_pack_and_batch():
    torch.manual_seed(0)
    x = torch.randn(4, 96, 500, device="cuda")       # (B, Cin, L): conv1d-style input
    w = torch.randn(160, 96, device="cuda")
    # Y_b^T (L, Cout) = X_b^T (L, Cin) @ W^T : A rows = L, k = Cin, element (l, ci) at x[b, ci, l]
    ap = ops.pack_split(x, 500, 96, 1, 500, 2, batch=4, batch_stride=96 * 500)
    bp = ops.pack_split(w, 160, 96, 96, 1, 2)
    y = ops.gemm_nt(ap, bp, 500, 160)
    ref = torch.einsum("bcl,oc->blo", x.double(), w.double())
    scale = torch.einsum("bcl,oc->blo", x.double().abs(), w.double().abs()).max()
    assert ((y.double() - ref).abs().max() / scale).item() < TOL[2]
    # batched B as well (attention-style): C[b] = A[b] @ B[b]^T
    a = torch.randn(3, 200, 64, device="cuda")
    b = torch.randn(3, 150, 64, device="cuda")
    ap = ops.pack_split(a, 200, 64, 64, 1, 2, batch=3, batch_stride=200 * 64)
    bp = ops.pack_split(b, 150, 64, 64, 1, 2, batch=3, batch_stride=150 * 64)
    c = ops.gemm_nt(ap, bp, 200, 150)
    ref = torch.bmm(a.double(), b.double().transpose(1, 2))
    assert ((c.double() - ref).abs().max() / 64).item() < 1e-4


def test_gemm_fp16_operands():
    torch.manual_seed(1)
    a = (torch.randn(1, 1, 256, 768, device="cuda") * 0.5).half()
    b = (torch.randn(1, 1, 3072, 768, device="cuda") * 0.05).half()
    c = ops.gemm_nt(a, b, 256, 3072)[0]
    ref = a[0, 0].double() @ b[0, 0].double().t()
    assert ((c.double() - ref).abs().max() / ref.abs().max()).item() < 2e-3


def test_gemm_split_k_weight_gradient_shape():
    """few output tiles, very long contraction (dW = dY^T X over a million rows) -> split-K path"""
    torch.manual_seed(2)
    m, n, k = 200000, 128, 64
    x = torch.randn(m, k, device="cuda")
    dy = torch.randn(m, n, device="cuda")
    dyt = ops.pack_split(dy, n, m, 1, n, 3)
    xt = ops.pack_split(x, k, m, 1, k, 3)
    dw = ops.gemm_nt(dyt, xt, n, k)[0]
    ref = dy.double().t() @ x.double()
    assert ((dw.double() - ref).abs().max() / ref.abs().max()).item() < 1e-5
    # the splits' partial tiles are added in a fixed order: the same bits on every call
    assert torch.equal(ops.gemm_nt(dyt, xt, n, k)[0], dw)


def test_gemm_split_k_after_a_larger_split_k_launch():
    """The split-K scratch is shared: a larger launch first leaves non-zero partial tiles in it.  A shape whose
    k-blocks do not divide evenly among the splits (9 output tiles over 16384 contraction columns) must still read
    only the partials it wrote itself."""
    torch.manual_seed(3)
    x = torch.randn(200000, 64, device="cuda")
    dy = torch.randn(200000, 128, device="cuda")
    ops.gemm_nt(ops.pack_split(dy, 128, 200000, 1, 128, 3), ops.pack_split(x, 64, 200000, 1, 64, 3), 128, 64)
    m, n, k = 384, 384, 16384
    a = torch.randn(m, k, device="cuda")
    b = torch.randn(n, k, device="cuda")
    c = ops.gemm_nt(ops.pack_split(a, m, k, k, 1, 3), ops.pack_split(b, n, k, k, 1, 3), m, n)[0]
    ref = a.double() @ b.double().t()
    assert ((c.double() - ref).abs().max() / ref.abs().max()).item() < 1e-5


def test_linear_autograd_matches_torch():
    torch.manual_seed(3)
    x = torch.randn(3000, 256, device="cuda", requires_grad=True)
    w = (torch.randn(512, 256, device="cuda") * 0.05).requires_grad_(True)
    b = torch.randn(512, device="cuda", requires_grad=True)
    for relu in (False, True):
        y = ops.linear(x, w, b, relu=relu)
        ref = torch.nn.functional.linear(x.double(), w.double(), b.double())
        ref = ref.relu() if relu else ref
        torch.testing.assert_close(y.double(), ref, rtol=1e-5, atol=1e-5)
        g = torch.randn_like(y)
        gx, gw, gb = torch.autograd.grad(y, (x, w, b), g)
        rx, rw, rb = torch.autograd.grad(ref, (x, w, b), g.double())
        for got, exp in ((gx, rx), (gw, rw), (gb, rb)):   # fp32 accumulation over up to 3000 terms
            assert ((got.double() - exp.double()).abs().max() / exp.abs().max()).item() < 3e-5


@pytest.mark.parametrize("mc,m,n", [(64, 128, 128), (1000, 128, 64), (3000, 512, 256), (200000, 256, 128), (77, 13, 3)])
def test_gemm_tn_mn_major_operands(mc, m, n):
    """C = A^T B from row-packed planes (MN-major tensor-core operands): the weight-gradient form"""
    torch.manual_seed(mc + m)
    a = torch.randn(mc, m, device="cuda")
    b = torch.randn(mc, n, device="cuda")
    ap = ops.pack_split(a, mc, m, m, 1, 3)
    bp = ops.pack_split(b, mc, n, n, 1, 3)
    c = ops.gemm_tn(ap, bp, m, n)
    ref = a.double().t() @ b.double()
    assert ((c.double() - ref).abs().max() / ref.abs().max()).item() < 2e-5


def test_gemm_fp16_output_and_quick_gelu():
    torch.manual_seed(5)
    x = (torch.randn(700, 768, device="cuda") * 0.5).half()
    w = (torch.randn(3072, 768, device="cuda") * 0.03).half()
    b = (torch.randn(3072, device="cuda") * 0.1).half()
    y = ops.linear(x, w, b, quick_gelu=True)
    assert y.dtype == torch.float16
    ref = torch.nn.functional.linear(x.double(), w.double(), b.double())
    ref = ref * torch.sigmoid(1.702 * ref)
    assert ((y.double() - ref).abs().max() / ref.abs().max()).item() < 2e-3
    y2 = ops.linear(x, w, None)
    ref2 = torch.nn.functional.linear(x.double(), w.double())
    assert ((y2.double() - ref2).abs().max() / ref2.abs().max()).item() < 2e-3


def test_fp16_linear_with_fused_residual_and_gelu():
    """CLIP block pattern: y = x_res + (QuickGELU?)(x W^T + b), residual added in the GEMM epilogue."""
    torch.manual_seed(5)
    m, k, n = 300, 768, 768          # ragged last row tile
    x = (torch.randn(m, k, device="cuda") * 0.2).half()
    w = (torch.randn(n, k, device="cuda") * 0.05).half()
    b = (torch.randn(n, device="cuda") * 0.1).half()
    res = torch.randn(m, n, device="cuda").half()
    for gelu in (False, True):
        y = ops.linear(x, w, b, quick_gelu=gelu, residual=res)
        lin = x.double() @ w.double().t() + b.double()
        if gelu:
            lin = lin * torch.sigmoid(1.702 * lin)
        ref = lin + res.double()
        assert y.dtype == torch.float16 and y.shape == (m, n)
        assert ((y.double() - ref).abs().max() / ref.abs().max()).item() < 2e-3     # fp16 output rounding
    # 3-D input / residual (L, N, D) as the tower passes them
    x3, r3 = x.view(50, 6, k), res.view(50, 6, n)
    assert torch.equal(ops.linear(x3, w, b, residual=r3).view(m, n), ops.linear(x, w, b, residual=res))


# ---------------------------------------------------------------- every instance, tile edges, split-K epilogue
# (nsplit, fp16, batch, m, n, k, bias, relu, ldc_pad): tests/test_gemm_instances_cpu.py checks that these reach every
# instance coda_gemm_nt can select and both sides of its split-K rule.  Output rows are ldc = n + ldc_pad apart.
NT_CASES = [
    # m, n, k at 1 and on either side of 64 and 128, on every fp32-plane instance
    (1, False, 1, 1, 1, 1, True, False, 0),
    (2, False, 1, 63, 65, 64, True, False, 3),
    (3, False, 1, 64, 63, 65, False, True, 0),
    (1, False, 1, 65, 64, 63, True, True, 1),
    (2, False, 1, 127, 129, 128, False, False, 4),
    (3, False, 1, 128, 127, 129, True, False, 0),
    (1, False, 1, 129, 128, 127, False, False, 2),
    (2, False, 1, 1, 64, 129, True, True, 0),
    (3, False, 1, 129, 1, 1, True, False, 5),
    # fp16 operands: 64-, 128-, 192- and 256-wide tiles, n = 512 below the 256-wide threshold
    (1, True, 1, 65, 1, 64, True, False, 0),
    (1, True, 1, 64, 64, 127, True, True, 3),
    (1, True, 1, 129, 65, 128, True, False, 0),
    (1, True, 1, 300, 512, 192, True, False, 4),
    (1, True, 1, 100, 1000, 64, False, False, 0),
    (1, True, 1, 200, 384, 64, True, False, 0),
    (1, True, 1, 130, 1536, 128, True, True, 0),
    # split-K: the bias, the batch index and ldc > n are handled by splitk_reduce_kernel, not the GEMM epilogue
    (1, False, 2, 129, 65, 4096, True, False, 3),
    (2, False, 3, 100, 64, 2100, True, False, 4),
    (3, False, 1, 200, 300, 8192, True, False, 0),
    (1, True, 2, 64, 200, 4096, True, False, 8),
    # a long contraction with ReLU never splits
    (2, False, 1, 100, 64, 4096, True, True, 0),
]

# exact fp16 operands: only the fp32 accumulation errs, as with three planes
FP16_TOL = TOL[3]
SENTINEL = 1234.5


def _nt_operand(x, nsplit, fp16):
    """(batch, rows, k) fp32 -> planes (nsplit, batch, rows, kpad): split bf16 planes, or one zero-padded fp16 plane"""
    batch, rows, k = x.shape
    if fp16:
        p = torch.zeros(1, batch, rows, ops._pad64(k), dtype=torch.float16, device=x.device)
        p[0, :, :, :k] = x.half()
        return p
    return ops.pack_split(x, rows, k, k, 1, nsplit, batch=batch, batch_stride=rows * k)


@pytest.mark.parametrize("nsplit,fp16,batch,m,n,k,bias,relu,ldc_pad", NT_CASES)
def test_gemm_nt_instances_and_edges_vs_fp64(nsplit, fp16, batch, m, n, k, bias, relu, ldc_pad):
    torch.manual_seed(7 * m + 3 * n + k + batch)
    a = torch.randn(batch, m, k, device="cuda")
    b = torch.randn(batch if batch == 3 else 1, n, k, device="cuda")      # batch 3: per-entry B, else shared weights
    if fp16:
        a, b = a.half().float(), b.half().float()
    bvec = torch.randn(n, device="cuda") if bias else None
    ap, bp = _nt_operand(a, nsplit, fp16), _nt_operand(b, nsplit, fp16)
    full = torch.full((batch, m, n + ldc_pad), SENTINEL, device="cuda")
    c = ops.gemm_nt(ap, bp, m, n, bias=bvec, relu=relu, out=full[..., :n])
    ref = _ref(a, b, bvec, relu)
    scale = (a.double().abs() @ b.double().abs().transpose(-1, -2)).max()
    err = ((c.double() - ref).abs().max() / scale).item()
    assert err < (FP16_TOL if fp16 else TOL[nsplit]), f"err {err:.2e}"
    assert bool((full[..., n:] == SENTINEL).all()), "a column >= n of the strided output was written"
    again = ops.gemm_nt(ap, bp, m, n, bias=bvec, relu=relu)
    assert torch.equal(again, c)


# (nsplit, mc, m, n): C (m, n) = A^T B over mc rows.  The 2- and 3-row outputs are the prediction heads' weight
# gradients (n_out = 2 / 3 rows, one per output feature), which run here on two planes.
TN_CASES = [
    (1, 1, 64, 64),
    (1, 65, 130, 129),
    (2, 1, 3, 2),
    (2, 65, 2, 256),
    (2, 4100, 3, 256),
    (2, 4100, 128, 3),
    (2, 3000, 130, 200),
    (2, 200000, 64, 64),
    (3, 65, 63, 65),
    (3, 200000, 128, 48),
]


def _tn(nsplit, mc, m, n, seed):
    torch.manual_seed(seed)
    a = torch.randn(mc, m, device="cuda")
    b = torch.randn(mc, n, device="cuda")
    return a, b, ops.pack_split(a, mc, m, m, 1, nsplit), ops.pack_split(b, mc, n, n, 1, nsplit)


@pytest.mark.parametrize("nsplit,mc,m,n", TN_CASES)
def test_gemm_tn_instances_and_edges_vs_fp64(nsplit, mc, m, n):
    a, b, ap, bp = _tn(nsplit, mc, m, n, mc + 5 * m + n)
    c = ops.gemm_tn(ap, bp, m, n)
    ref = a.double().t() @ b.double()
    scale = (a.double().abs().t() @ b.double().abs()).max()
    err = ((c.double() - ref).abs().max() / scale).item()
    assert err < TOL[nsplit], f"err {err:.2e}"


def test_gemm_tn_same_bits_after_a_larger_split_k_launch():
    """The heads' weight-gradient shape splits K; a larger split-K launch in between leaves its partial tiles in the
    shared scratch.  The second call must give the same bits."""
    _, _, ap, bp = _tn(2, 4100, 3, 256, 11)
    c1 = ops.gemm_tn(ap, bp, 3, 256)
    _, _, bigp, bigq = _tn(2, 200000, 256, 128, 12)
    ops.gemm_tn(bigp, bigq, 256, 128)
    assert torch.equal(ops.gemm_tn(ap, bp, 3, 256), c1)
