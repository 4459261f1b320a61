"""Fused wgmma attention forward against a float64 softmax(QK^T)V of the same inputs."""
import pytest
import torch

from coda_neurips2023_b200 import attention_launch, attention_sm100

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


def _ref64(q, k, v, nhead, keep=None, p=0.0):
    return attention_sm100._math(q.double(), k.double(), v.double(), nhead, p, False, False, keep)


CASES = [
    # lq, lk, b, heads, hd
    (128, 64, 1, 1, 64), (128, 128, 2, 2, 64), (2048, 2048, 2, 4, 64), (256, 256, 2, 4, 128),
    (256, 2048, 2, 4, 128), (100, 77, 3, 2, 64), (50, 50, 5, 12, 64), (130, 200, 1, 4, 128), (1, 1, 1, 1, 64),
]


NSPLIT_TOLS = [(3, 5e-6), (2, 1e-4), (1, 2e-2)]


@pytest.mark.parametrize("nsplit,tol", NSPLIT_TOLS)
@pytest.mark.parametrize("lq,lk,b,h,hd", CASES)
def test_attention_forward_vs_fp64(lq, lk, b, h, hd, nsplit, tol):
    torch.manual_seed(lq + lk + hd)
    e = h * hd
    q = torch.randn(lq, b, e, device="cuda") * 1.5
    k = torch.randn(lk, b, e, device="cuda") * 1.5
    v = torch.randn(lk, b, e, device="cuda")
    out, lse = attention_launch.forward(q, k, v, h, nsplit=nsplit)
    ref = _ref64(q, k, v, h)
    err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    assert err < tol, f"nsplit={nsplit}: rel err {err:.2e}"
    s = torch.einsum("qbhd,kbhd->bhqk", (q.double() * hd ** -0.5).view(lq, b, h, hd), k.double().view(lk, b, h, hd))
    ref_lse = torch.logsumexp(s, dim=-1).reshape(b * h, lq)
    assert (lse.double() - ref_lse).abs().max().item() < max(tol * 50, 1e-5)


def test_attention_dropout_mask_matches_torch_twin():
    torch.manual_seed(0)
    lq, lk, b, h, hd = 256, 320, 2, 4, 64
    q, k, v = (torch.randn(n, b, h * hd, device="cuda") for n in (lq, lk, lk))
    attention_launch.seed_counter(q.device).fill_(12345)
    out, _ = attention_launch.forward(q, k, v, h, dropout_p=0.1, salt=777, nsplit=3)
    keep = attention_launch.dropout_keep(b * h, lq, lk, 0.1, 777, q.device)
    assert 0.88 < keep.float().mean().item() < 0.92
    mult = attention_launch.dropout_mult(b * h, lq, lk, 0.1, 777, q.device)
    assert torch.equal(mult > 0, keep) and abs(mult.max().item() - 1 / 0.9) < 1e-6
    ref = _ref64(q, k, v, h, keep, 0.1)
    assert ((out.double() - ref).abs().max() / ref.abs().max()).item() < 5e-6


def test_attention_autograd_wrapper():
    torch.manual_seed(1)
    lq, lk, b, h, hd = 200, 300, 2, 4, 64
    q, k, v = (torch.randn(n, b, h * hd, device="cuda", requires_grad=True) for n in (lq, lk, lk))
    out = attention_sm100.attention(q, k, v, h)          # the step's default: two operand planes in the forward
    ref = attention_sm100._math(q, k, v, h, 0.0, False, False)
    torch.testing.assert_close(out, ref, rtol=1e-4, atol=2e-5)
    g = torch.randn_like(out)
    got = torch.autograd.grad(out, (q, k, v), g)
    exp = torch.autograd.grad(ref, (q, k, v), g)
    for a, e in zip(got, exp):
        torch.testing.assert_close(a, e, rtol=1e-4, atol=1e-5)
    # training-mode dropout goes through the kernel + regenerated mask and stays unbiased
    outs = torch.stack([attention_sm100.attention(q, k, v, h, 0.1, True).detach() for _ in range(8)])
    assert (outs.mean(0) - ref.detach()).abs().mean().item() < 0.05


BWD_CASES = [
    (128, 128, 1, 1, 64), (2048, 2048, 1, 4, 64), (300, 200, 2, 2, 64), (64, 1000, 2, 4, 64), (50, 50, 3, 12, 64),
    (128, 64, 1, 1, 128), (256, 2048, 2, 4, 128), (256, 256, 2, 4, 128), (130, 200, 1, 2, 128), (3, 2, 1, 1, 128)]


@pytest.mark.parametrize("lq,lk,b,h,hd", BWD_CASES)
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_attention_backward_vs_fp64(lq, lk, b, h, hd, p):
    torch.manual_seed(lq + lk)
    e = h * hd
    q = (torch.randn(lq, b, e, device="cuda") * 1.2).requires_grad_(True)
    k = (torch.randn(lk, b, e, device="cuda") * 1.2).requires_grad_(True)
    v = torch.randn(lk, b, e, device="cuda", requires_grad=True)
    attention_launch.seed_counter(q.device).fill_(4242)
    out, lse = attention_launch.forward(q.detach(), k.detach(), v.detach(), h, dropout_p=p, salt=99, nsplit=3)
    g = torch.randn_like(out)
    dq, dk, dv = attention_launch.backward(q.detach(), k.detach(), v.detach(), out, g, lse, h, p, 99)
    keep = attention_launch.dropout_keep(b * h, lq, lk, p, 99, q.device) if p > 0 else None
    q64, k64, v64 = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = attention_sm100._math(q64, k64, v64, h, p, False, False, keep)
    rq, rk, rv = torch.autograd.grad(ref, (q64, k64, v64), g.double())
    for name, got, exp in (("dq", dq, rq), ("dk", dk, rk), ("dv", dv, rv)):
        err = ((got.double() - exp).abs().max() / exp.abs().max()).item()
        assert err < 2e-4, f"{name}: rel err {err:.2e}"


def test_attention_forward_reads_fp16_slices_of_a_fused_projection_in_place():
    """CLIP tower call pattern: q, k, v are fp16 column slices of one (L, B, 3E) tensor; the pack kernel reads them
    strided and as half.  Must equal the kernel run on contiguous fp32 copies of the same values bit for bit."""
    torch.manual_seed(3)
    l, b, h = 50, 7, 12
    e = h * 64
    qkv = (torch.randn(l, b, 3 * e, device="cuda") * 0.7).half()
    q, k, v = qkv.split(e, dim=-1)
    assert not q.is_contiguous()
    out_h, lse_h = attention_launch.forward(q, k, v, h, nsplit=2)
    out_f, lse_f = attention_launch.forward(q.float().contiguous(), k.float().contiguous(), v.float().contiguous(), h, nsplit=2)
    assert out_h.dtype == torch.float32 and torch.equal(out_h, out_f) and torch.equal(lse_h, lse_f)
    # fp16 output straight from the kernel (single-tile instance) = the fp32 result rounded once
    out_16, _ = attention_launch.forward(q, k, v, h, nsplit=2, half_out=True)
    assert out_16.dtype == torch.float16 and torch.equal(out_16, out_h.half())
    # and an fp32 strided slice (encoder-style fused projection)
    qkv32 = torch.randn(130, 2, 3 * 256, device="cuda")
    q2, k2, v2 = qkv32.split(256, dim=-1)
    o_s, _ = attention_launch.forward(q2, k2, v2, 4)
    o_c, _ = attention_launch.forward(q2.contiguous(), k2.contiguous(), v2.contiguous(), 4)
    assert torch.equal(o_s, o_c)


MASKED_CASES = [(256, 256, 2, 4, 64), (2048, 2048, 1, 4, 64), (130, 200, 2, 2, 64), (256, 2048, 2, 4, 128),
                (100, 77, 1, 2, 128)]


@pytest.mark.parametrize("lq,lk,b,h,hd", MASKED_CASES)
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_masked_attention_forward_backward_vs_fp64(lq, lk, b, h, hd, p):
    """Boolean attn_mask (True = not visible; nn.MultiheadAttention's convention, the reference's masked encoder
    transformer.py:146-211) applied inside the fused kernels, forward and backward, against the fp64 formula.  The
    masks include rows whose first key tiles are entirely masked (running max stays -inf for a while)."""
    torch.manual_seed(lq * 3 + lk)
    e = h * hd
    q = torch.randn(lq, b, e, device="cuda") * 1.2
    k = torch.randn(lk, b, e, device="cuda") * 1.2
    v = torch.randn(lk, b, e, device="cuda")
    mask = torch.rand(b, lq, lk, device="cuda") < 0.6
    mask[:, : lq // 2, : min(lk, 192) // 2] = True             # leading key tiles fully masked for half the rows
    mask[:, :, lk - 1] = False                                 # every row keeps at least one key
    bits = attention_launch.mask_bits(mask, b)
    attention_launch.seed_counter(q.device).fill_(77)
    out, lse = attention_launch.forward(q, k, v, h, dropout_p=p, salt=5, mask=bits, nsplit=3)
    g = torch.randn_like(out)
    dq, dk, dv = attention_launch.backward(q, k, v, out, g, lse, h, p, 5, mask=bits)
    keep = attention_launch.dropout_keep(b * h, lq, lk, p, 5, q.device) if p > 0 else None
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref = attention_sm100._math(q64, k64, v64, h, p, False, False, keep, attn_mask=mask)
    assert torch.isfinite(out).all()
    assert ((out.double() - ref).abs().max() / ref.abs().max()).item() < 5e-6
    rq, rk, rv = torch.autograd.grad(ref, (q64, k64, v64), g.double())
    for name, got, exp in (("dq", dq, rq), ("dk", dk, rk), ("dv", dv, rv)):
        err = ((got.double() - exp).abs().max() / exp.abs().max()).item()
        assert err < 2e-4, f"{name}: rel err {err:.2e}"


def test_radius_mask_bits_equal_cdist_mask():
    """The packed radius mask built from coordinates == packing the reference's `cdist(xyz, xyz) >= radius`
    (points exactly on the threshold aside: none in this draw), and broadcast / per-scene packing agree."""
    torch.manual_seed(4)
    xyz = torch.rand(3, 1000, 3, device="cuda") * 3
    radius = 0.4 ** 2 * 4
    dense = torch.cdist(xyz.double(), xyz.double()) >= radius
    bq, bk = attention_launch.radius_mask_bits(xyz, radius)
    eq, ek = attention_launch.mask_bits(dense, 3)
    assert bq is bk and torch.equal(bq, eq) and torch.equal(bk, ek)
    one = attention_launch.mask_bits(dense[0], 3)          # (Lq, Lk) mask broadcast over the batch
    assert torch.equal(one[0][1], eq[0]) and torch.equal(one[1][2], ek[0])


def test_fused_projection_layouts_match_separate_tensors():
    """attention_fused ("qkv" / "qk_v": slices of ONE projection read in place, ONE packed gradient written by the
    backward) == the three-tensor call on copies, values and gradients bit for bit."""
    torch.manual_seed(6)
    l, b, h, e = 300, 2, 4, 256
    for layout in ("qkv", "qk_v"):
        width = 3 * e if layout == "qkv" else 2 * e
        a = torch.randn(l, b, width, device="cuda", requires_grad=True)
        vsep = torch.randn(l, b, e, device="cuda", requires_grad=True) if layout == "qk_v" else None
        out = attention_sm100.attention_fused(a, vsep, layout, h)
        g = torch.randn_like(out)
        grads = torch.autograd.grad(out, (a,) if vsep is None else (a, vsep), g)
        parts = [a.detach()[..., i * e: (i + 1) * e].clone().requires_grad_(True) for i in range(width // e)]
        if vsep is not None:
            parts.append(vsep.detach().clone().requires_grad_(True))
        ref = attention_sm100.attention(parts[0], parts[1], parts[2], h)
        rg = torch.autograd.grad(ref, parts, g)
        assert torch.equal(out, ref)
        assert grads[0].is_contiguous() and torch.equal(grads[0], torch.cat(rg[: width // e], dim=-1))
        if vsep is not None:
            assert torch.equal(grads[1], rg[2])


def test_half_operand_attention_of_the_clip_tower():
    """coda_attention_fwd_half: fp16 q / k / v slices of a fused projection, ONE plane of half operands (no bf16
    split), fp16 output -- against the fp32 formula on the same half values.  fp16 probabilities carry 11 mantissa
    bits (like the reference, whose nn.MultiheadAttention runs entirely in half): 2e-3."""
    torch.manual_seed(8)
    l, b, h = 50, 37, 12
    e = h * 64
    qkv = (torch.randn(l, b, 3 * e, device="cuda") * 0.8).half()
    q, k, v = qkv.split(e, dim=-1)
    out = attention_launch.forward_half(q, k, v, h)
    assert out.dtype == torch.float16 and out.shape == (l, b, e)
    ref = attention_sm100._math(q.float(), k.float(), v.float(), h, 0.0, False, False)
    assert ((out.float() - ref).abs().max() / ref.abs().max()).item() < 2e-3
    # contiguous inputs take the same path
    out2 = attention_launch.forward_half(q.contiguous(), k.contiguous(), v.contiguous(), h)
    assert torch.equal(out, out2)


def test_default_forward_split_is_two_planes_and_meets_1e4():
    """attention_launch.FORWARD_NSPLIT (2 unless CODA_ATTN_NSPLIT overrides it): the default call equals the explicit
    two-plane call bit for bit and sits within 1e-4 of the fp64 formula on the encoder and decoder shapes."""
    torch.manual_seed(11)
    for lq, lk, b, h, hd in ((2048, 2048, 1, 4, 64), (256, 2048, 2, 4, 128)):
        e = h * hd
        q = torch.randn(lq, b, e, device="cuda") * 1.5
        k = torch.randn(lk, b, e, device="cuda") * 1.5
        v = torch.randn(lk, b, e, device="cuda")
        out, _ = attention_launch.forward(q, k, v, h)
        if attention_launch.FORWARD_NSPLIT == 2:
            assert torch.equal(out, attention_launch.forward(q, k, v, h, nsplit=2)[0])
        ref = _ref64(q, k, v, h)
        assert ((out.double() - ref).abs().max() / ref.abs().max()).item() < 1e-4
