"""GPU tests of the step-glue kernels (include/coda_step.h) against plain PyTorch fp32 references, and of
engine.TrainStep's bookkeeping (probe / restore, inactive parameters, parameter groups)."""
import copy
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def test_dropout_add_mask_is_shared_by_forward_and_backward():
    from coda_neurips2023_b200 import attention_launch, ops

    torch.manual_seed(0)
    x = torch.randn(2048, 8, 256, device="cuda")
    x = x.masked_fill(x == 0, 1.0).requires_grad_()   # the mask is read off delta / x below: no exact zeros in x
    r = torch.randn_like(x, requires_grad=True)
    attention_launch.advance_seed(x.device)
    out = ops.dropout_add(x, r, 0.1, True)
    delta = (out - r).detach()                         # x * (0 or 1 / 0.9) up to the rounding of the addition
    keep = (delta / x.detach()) > 0.5
    mult = keep.float() / 0.9
    assert torch.allclose(delta, x.detach() * mult, rtol=1e-5, atol=2e-6)
    frac = keep.float().mean().item()
    assert abs(frac - 0.9) < 2e-3, frac
    g = torch.randn_like(out)
    out.backward(g)
    assert torch.equal(r.grad, g)
    assert torch.allclose(x.grad, g * mult, rtol=1e-6, atol=1e-7)
    # a second call site draws a different mask, the next step (advanced seed) too
    out2 = ops.dropout_add(x, r, 0.1, True)
    assert ((out2 - r) / x > 0.5).ne(keep).any()
    # p = 0 / eval: exact add, odd length exercises the scalar tail
    a, b = torch.randn(1027, device="cuda"), torch.randn(1027, device="cuda")
    assert torch.equal(ops.dropout_add(a, b, 0.3, False), a + b)
    d = ops.dropout(a, 0.5, True)
    assert ((d == 0) | torch.isclose(d, a * 2)).all() and 0.4 < (d != 0).float().mean().item() < 0.6


@pytest.mark.parametrize("rows,c,relu", [(16384, 512, True), (1000, 64, True), (777, 256, False)])
def test_bn_act_rows_matches_torch(rows, c, relu):
    from coda_neurips2023_b200 import ops

    torch.manual_seed(1)
    bn = torch.nn.BatchNorm1d(c).cuda().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.2)
    ref_bn = copy.deepcopy(bn)
    h = (torch.randn(rows, c, device="cuda") * 1.7 + 0.3).requires_grad_(True)
    h2 = h.detach().clone().requires_grad_(True)
    out = ops.bn_act_rows(h, bn, relu, 0.0, True)
    exp = ref_bn(h2)
    exp = torch.relu(exp) if relu else exp
    assert torch.allclose(out, exp, rtol=1e-5, atol=2e-6)
    assert torch.allclose(bn.running_mean, ref_bn.running_mean, rtol=1e-5, atol=1e-6)
    assert torch.allclose(bn.running_var, ref_bn.running_var, rtol=1e-5, atol=1e-6)
    assert int(bn.num_batches_tracked) == 1
    g = torch.randn_like(out)
    out.backward(g)
    exp.backward(g)
    scale = h2.grad.abs().max()
    assert (h.grad - h2.grad).abs().max() <= 2e-5 * scale
    assert torch.allclose(bn.weight.grad, ref_bn.weight.grad, rtol=1e-4, atol=1e-4 * ref_bn.weight.grad.abs().max().item())
    assert torch.allclose(bn.bias.grad, ref_bn.bias.grad, rtol=1e-4, atol=1e-4 * ref_bn.bias.grad.abs().max().item())
    # eval mode: running statistics
    bn.eval(); ref_bn.eval()
    with torch.no_grad():
        o, e = ops.bn_act_rows(h, bn, relu, 0.3, False), ref_bn(h)
    assert torch.allclose(o, torch.relu(e) if relu else e, rtol=1e-5, atol=1e-5)


def test_bn_act_rows_dropout_backward_consistent():
    from coda_neurips2023_b200 import attention_launch, ops

    torch.manual_seed(2)
    bn = torch.nn.BatchNorm1d(512).cuda().train()
    h = torch.randn(4096, 512, device="cuda", requires_grad=True)
    attention_launch.advance_seed(h.device)
    out = ops.bn_act_rows(h, bn, True, 0.3, True)
    plain = torch.relu(torch.nn.functional.batch_norm(h.detach(), None, None, bn.weight, bn.bias, True))
    pos = plain > 1e-3
    mult = (out.detach() / plain)[pos]
    assert ((mult - 1 / 0.7).abs() < 1e-4).logical_or(mult.abs() < 1e-6).all()
    keepfrac = (mult > 0.5).float().mean().item()
    assert abs(keepfrac - 0.7) < 5e-3
    # backward == autograd through the same mask
    mask = torch.zeros_like(plain)
    mask[pos] = mult
    mask[~pos] = (out.detach()[~pos] != 0).float() / 0.7
    h2 = h.detach().clone().requires_grad_(True)
    ref = torch.relu(torch.nn.functional.batch_norm(h2, None, None, bn.weight, bn.bias, True)) * mask
    g = torch.randn_like(out)
    out.backward(g)
    ref.backward(g)
    assert (h.grad - h2.grad).abs().max() <= 5e-5 * h2.grad.abs().max()


@pytest.mark.parametrize("filter_biases", [False, True])
def test_flat_adamw_matches_torch_adamw_with_clip(filter_biases):
    from coda_neurips2023_b200.engine import FlatAdamW, FlatParameters, _no_decay

    torch.manual_seed(3)
    # odd sizes and one tensor longer than a chunk; FlatParameters starts every tensor on a 64-element boundary, so
    # the chunk offsets are multiples of 4 here (test_step_glue_edges_gpu.py runs unaligned chunk tables)
    model = torch.nn.Sequential(torch.nn.Linear(37, 501), torch.nn.ReLU(), torch.nn.Linear(501, 129),
                                torch.nn.LayerNorm(129), torch.nn.Linear(129, 7)).cuda()
    ref = copy.deepcopy(model)
    flat = FlatParameters(model)
    lr = torch.tensor(3e-3, device="cuda")
    wds = [0.0 if (filter_biases and _no_decay(n, p)) else 0.1 for n, p in zip(flat.names, flat.params)]
    opt = FlatAdamW(flat, lr, wds, max_norm=0.1)
    decay = [p for n, p in ref.named_parameters() if not (filter_biases and _no_decay(n, p))]
    nodecay = [p for n, p in ref.named_parameters() if filter_biases and _no_decay(n, p)]
    groups = [{"params": decay, "weight_decay": 0.1}] + ([{"params": nodecay, "weight_decay": 0.0}] if nodecay else [])
    topt = torch.optim.AdamW(groups, lr=3e-3)
    for it in range(5):
        x = torch.randn(64, 37, device="cuda")
        flat.zero_grad()
        model(x).pow(2).mean().backward()
        opt.step()
        topt.zero_grad()
        ref(x).pow(2).mean().backward()
        norm = torch.nn.utils.clip_grad_norm_(ref.parameters(), 0.1)
        topt.step()
        assert abs(float(opt.grad_norm) - float(norm)) <= 1e-5 * float(norm)
        for p, q in zip(model.parameters(), ref.parameters()):
            assert torch.allclose(p, q, rtol=2e-5, atol=2e-7), it


def test_flat_adamw_leaves_inactive_parameters_alone():
    from coda_neurips2023_b200.engine import FlatAdamW, FlatParameters

    torch.manual_seed(4)
    model = torch.nn.ModuleDict({"used": torch.nn.Linear(8, 8), "unused": torch.nn.Linear(8, 8)}).cuda()
    before = model["unused"].weight.detach().clone()
    flat = FlatParameters(model)
    active = [n.startswith("used") for n in flat.names]
    opt = FlatAdamW(flat, torch.tensor(1e-2, device="cuda"), 0.1, active)
    flat.zero_grad()
    model["used"](torch.randn(4, 8, device="cuda")).sum().backward()
    opt.step()
    assert torch.equal(model["unused"].weight, before)          # no weight decay on a parameter without gradient
    assert not torch.equal(model["used"].weight, flat.flat_param.data.new_zeros(8, 8))


def test_train_step_prepare_and_capture_leave_no_trace():
    """ADVICE r1: probe + graph warm-up must not advance the optimizer, BatchNorm buffers or the dropout counter;
    parameters without gradient (text head when its loss weight is 0) are not decayed; the step is deterministic
    given the same state, eager == captured graph."""
    from coda_neurips2023_b200 import attention_launch, synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.engine import TrainStep
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(nqueries=128, preenc_npoints=256, dec_dim=128, dec_nlayers=2, dec_ffn_dim=64,
                               enc_dropout=0.0, dec_dropout=0.0, mlp_dropout=0.0,   # call-site salts differ eager/graph
                               loss_predicted_region_embed_l1_weight=0.0, filter_biases_wd=True)
    cfg = synthetic.SyntheticDatasetConfig(args)

    def make():
        torch.manual_seed(0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = build_model(args, cfg)
        return model.cuda().train(), build_criterion(args, cfg).cuda()

    batch = synthetic.to_device(synthetic.make_batch(2, 3000, seed=1), "cuda")
    model, crit = make()
    w0 = {n: p.detach().clone() for n, p in model.named_parameters() if p.requires_grad}
    bn0 = {n: b.detach().clone() for n, b in model.named_buffers() if "clip_model" not in n}
    seed0 = int(attention_launch.seed_counter(torch.device("cuda", 0)))
    step = TrainStep(args, model, crit, torch.device("cuda", 0))
    np.random.seed(11)
    step.capture(batch, warmup=2)
    assert int(step.optimizer.state[0]) == 0, "warm-up advanced the optimizer"
    assert int(attention_launch.seed_counter(torch.device("cuda", 0))) == seed0
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert torch.equal(p, w0[n]), n
    for n, b in model.named_buffers():
        if "clip_model" not in n:
            assert torch.equal(b, bn0[n]), n
    assert any("text_correlation_head" in n for n in step.inactive_names)
    np.random.seed(12)
    loss_g, _ = step(batch, 0.0)
    loss_g = float(loss_g)
    assert int(step.optimizer.state[0]) == 1
    for n, p in model.named_parameters():
        if "text_correlation_head" in n:
            assert torch.equal(p, w0[n]), f"{n} was decayed without a gradient"
    wg = {n: p.detach().clone() for n, p in model.named_parameters() if p.requires_grad}
    # the same step eagerly from the same initial state
    model2, crit2 = make()
    attention_launch.seed_counter(torch.device("cuda", 0)).fill_(seed0)
    step2 = TrainStep(args, model2, crit2, torch.device("cuda", 0))
    step2.prepare(batch)
    np.random.seed(12)
    loss_e, _ = step2(batch, 0.0)
    assert abs(float(loss_e) - loss_g) <= 1e-5 * abs(loss_g)
    changed = 0
    for n, p in model2.named_parameters():
        if p.requires_grad:
            assert torch.allclose(p, wg[n], rtol=1e-4, atol=1e-6), n
            changed += int(not torch.equal(p, w0[n]))
    assert changed > 100


# ------------------------------------------------------------------ fused autograd joins (round 2)
def _ln_ref(x, w, b, eps=1e-5):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), w, b, eps)


@pytest.mark.parametrize("q,b,c,with_pos,want_y", [(256, 8, 512, True, True), (256, 8, 512, True, False),
                                                   (100, 3, 256, False, True), (2048, 8, 256, False, True)])
def test_layer_norm_branch_matches_the_unfused_graph(q, b, c, with_pos, want_y):
    """(x, norm(x), norm(x) + pos) as one node == x / LayerNorm / add as three, values and every gradient (the
    residual by-pass gradient and the `+ pos` gradient are added inside the backward kernel)"""
    from coda_neurips2023_b200 import ops

    torch.manual_seed(q + c)
    norm = ops.LayerNorm(c).cuda()
    with torch.no_grad():
        norm.weight.normal_(1.0, 0.2)
        norm.bias.normal_(0.0, 0.2)
    x = torch.randn(q, b, c, device="cuda", requires_grad=True)
    pos = torch.randn(q, b, c, device="cuda", requires_grad=True) if with_pos else None
    x_id, y, yp = ops.layer_norm_branch(x, norm, pos, want_y=want_y)
    xr = x.detach().double().requires_grad_(True)
    pr = pos.detach().double().requires_grad_(True) if with_pos else None
    wr, br = norm.weight.detach().double().requires_grad_(True), norm.bias.detach().double().requires_grad_(True)
    yr = _ln_ref(xr, wr, br)
    ypr = yr + pr if with_pos else yr
    assert x_id.data_ptr() == x.data_ptr()
    # a strided input comes back as its contiguous copy (same values), not as a second strided operand
    xs = torch.randn(b, c, q, device="cuda").permute(2, 0, 1)
    xs_id, ys, _ = ops.layer_norm_branch(xs, norm)
    assert xs_id.is_contiguous() and torch.equal(xs_id, xs)
    torch.testing.assert_close(ys, _ln_ref(xs, norm.weight, norm.bias), rtol=1e-5, atol=1e-5)
    if want_y:
        torch.testing.assert_close(y.double(), yr, rtol=1e-5, atol=1e-5)
    else:
        assert y is None
    torch.testing.assert_close(yp.double(), ypr, rtol=1e-5, atol=1e-5)
    g1, g2, g3 = (torch.randn(q, b, c, device="cuda") for _ in range(3))
    loss = (x_id * g1).sum() + (yp * g3).sum() + ((y * g2).sum() if want_y and with_pos else 0.0)
    ref = (xr * g1.double()).sum() + (ypr * g3.double()).sum() + ((yr * g2.double()).sum() if want_y and with_pos else 0.0)
    ins = [x, norm.weight, norm.bias] + ([pos] if with_pos else [])
    rins = [xr, wr, br] + ([pr] if with_pos else [])
    got = torch.autograd.grad(loss, ins)
    exp = torch.autograd.grad(ref, rins)
    for gg, ee in zip(got, exp):
        assert ((gg.double() - ee).abs().max() / ee.abs().max()).item() < 2e-5


def test_norm_stack_writes_the_heads_layout_and_its_backward():
    """norm of every decoder layer's output straight into (layers, batch, query, channel): equals
    torch.stack([norm(x_l)]).permute(0, 2, 1, 3), gradients included (gamma / beta summed over the layers)"""
    from coda_neurips2023_b200 import ops

    torch.manual_seed(9)
    nl, q, b, c = 4, 96, 3, 256
    norm = ops.LayerNorm(c).cuda()
    with torch.no_grad():
        norm.weight.normal_(1.0, 0.2)
        norm.bias.normal_(0.0, 0.2)
    xs = [torch.randn(q, b, c, device="cuda", requires_grad=True) for _ in range(nl)]
    assert ops.norm_stack_applicable(norm, xs)
    out = ops.norm_stack(norm, xs)
    assert out.shape == (nl, b, q, c) and out.is_contiguous()
    xr = [x.detach().double().requires_grad_(True) for x in xs]
    wr, br = norm.weight.detach().double().requires_grad_(True), norm.bias.detach().double().requires_grad_(True)
    ref = torch.stack([_ln_ref(x, wr, br) for x in xr]).permute(0, 2, 1, 3)
    torch.testing.assert_close(out.double(), ref, rtol=1e-5, atol=1e-5)
    g = torch.randn(nl, b, q, c, device="cuda")
    got = torch.autograd.grad(out, [norm.weight, norm.bias, *xs], g)
    exp = torch.autograd.grad(ref, [wr, br, *xr], g.double())
    for gg, ee in zip(got, exp):
        assert ((gg.double() - ee).abs().max() / ee.abs().max()).item() < 2e-5


@pytest.mark.parametrize("n,count", [(8 * 256 * 512, 6), (1027, 3), (4096, 16), (4100, 21), (12, 1)])
def test_sum_tensors_and_fanout(n, count):
    from coda_neurips2023_b200 import ops

    torch.manual_seed(n)
    ts = [torch.randn(n, device="cuda") for _ in range(count)]
    ref = torch.stack([t.double() for t in ts]).sum(0)
    got = ops.sum_tensors(ts)
    assert ((got.double() - ref).abs().max() / ref.abs().max()).item() < 2e-6
    x = torch.randn(n, device="cuda", requires_grad=True)
    taps = ops.fanout(x, count)
    assert len(taps) == count and all(t.data_ptr() == x.data_ptr() for t in taps)
    loss = sum((t * w).sum() for t, w in zip(taps, ts))
    (gx,) = torch.autograd.grad(loss, x)
    assert ((gx.double() - ref).abs().max() / ref.abs().max()).item() < 2e-6
    # unused taps contribute nothing
    if count > 2:
        taps = ops.fanout(x, count)
        (gx,) = torch.autograd.grad((taps[0] * ts[0]).sum() + (taps[2] * ts[2]).sum(), x)
        torch.testing.assert_close(gx, ts[0] + ts[2])


@pytest.mark.parametrize("nl,b,q,d", [(7, 8, 256, 512), (1, 2, 50, 64)])
def test_masked_l1_matches_the_reference_expression(nl, b, q, d):
    """reference criterion.py:924-943: (pred * w - target * w).abs().sum over everything but the layer"""
    from coda_neurips2023_b200 import ops

    torch.manual_seed(nl)
    pred = torch.randn(nl, b, q, d, device="cuda", requires_grad=True)
    target = torch.randn(b, q, d, device="cuda")
    w = (torch.rand(b, q, 1, device="cuda") > 0.6).float()
    with torch.no_grad():
        pred[0, 0, 0, :8] = target[0, 0, :8]          # exact zeros: sgn(0) = 0
    out = ops.masked_l1(pred, target, w)
    pr = pred.detach().double().requires_grad_(True)
    ref = (pr * w.double() - target.double() * w.double()).abs().sum(dim=(1, 2, 3))
    assert ((out.double() - ref).abs() / ref).max().item() < 1e-6
    g = torch.rand(nl, device="cuda") + 0.5
    (got,) = torch.autograd.grad(out, pred, g)
    (exp,) = torch.autograd.grad(ref, pr, g.double())
    torch.testing.assert_close(got.double(), exp, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("m,k,n", [(16384, 256, 128), (2048, 512, 256), (3000, 256, 512), (2048, 512, 512)])
def test_linear_relu_backward_masks_inside_the_gemms(m, k, n):
    """y = relu(x W^T + b): the backward evaluates [y > 0] * dY in the A prologue of both gradient GEMMs -- same
    values as masking first (the fallback for shapes the prologue does not take)"""
    from coda_neurips2023_b200 import ops

    torch.manual_seed(m + n)
    x = torch.randn(m, k, device="cuda", requires_grad=True)
    w = (torch.randn(n, k, device="cuda") * 0.05).requires_grad_(True)
    b = torch.randn(n, device="cuda", requires_grad=True)
    y = ops.linear(x, w, b, relu=True)
    g = torch.randn_like(y)
    gx, gw, gb = torch.autograd.grad(y, (x, w, b), g)
    # the same backward on a pre-masked gradient through the plain (relu = False) node
    y0 = ops.linear(x, w, b, relu=False)
    gm = g * (y0.detach() > 0).float()
    rx, rw, rb = torch.autograd.grad(y0, (x, w, b), gm)
    # same operand values through the same tensor-core sequence; the split-K partition of the weight gradient may
    # differ between the two prologues (fp32 re-association): compare on the scale of the result
    for got, exp in ((gx, rx), (gw, rw)):
        assert ((got - exp).abs().max() / exp.abs().max()).item() < 2e-6
    torch.testing.assert_close(gb, rb, rtol=1e-5, atol=1e-4)
    # and against fp64 with the mask the forward produced (an fp64 forward flips the mask where y is within rounding
    # of zero, which is not an error of the backward)
    gd = gm.double()
    for got, exp in ((gx, gd @ w.detach().double()), (gw, gd.t() @ x.detach().double()), (gb, gd.sum(0))):
        assert ((got.double() - exp).abs().max() / exp.abs().max()).item() < 3e-5
