"""The decoder's cross-attention K / V bank (ops.kv_bank + MultiheadAttention.forward_bank) against a float64
restatement of the same layers: every layer's keys and values projected by one GEMM, attention reading its slice with
row stride nlayers * e, dK / dV written into slices of one shared gradient buffer, and one 4096-long contraction
adding up the input gradient of all layers."""
import pytest
import torch

from coda_neurips2023_b200 import attention_launch, attention_sm100, ops
from coda_neurips2023_b200.models.transformer import MultiheadAttention

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


def _rel(got, exp, scale=None):
    got = torch.zeros_like(exp) if got is None else got.detach().double()
    return float((got - exp).abs().max() / (exp.abs().max() if scale is None else scale))


def _poison_free_blocks(shape, count=4):
    """Leave NaN-filled blocks of `shape` in the caching allocator: a buffer allocated without a zero fill and
    not completely written then shows up as NaN instead of happening to read zeros."""
    blocks = [torch.full(shape, float("nan"), device="cuda") for _ in range(count)]
    del blocks


@pytest.mark.parametrize("nl,e,h,lk,b,lq,p,unused", [
    (2, 256, 4, 300, 2, 100, 0.0, None),
    (8, 512, 4, 2048, 2, 256, 0.0, None),      # the decoder of the training step
    (3, 256, 2, 300, 2, 100, 0.1, None),       # head dim 128, attention dropout
    (3, 256, 4, 300, 2, 100, 0.0, 1),          # layer 1's output does not reach the loss
])
def test_kv_bank_matches_fp64_layers(monkeypatch, nl, e, h, lk, b, lq, p, unused):
    torch.manual_seed(nl * 1000 + e + lk)
    mods = []
    for _ in range(nl):
        m = MultiheadAttention(e, h, dropout=p).cuda().train()
        with torch.no_grad():
            m.in_proj_bias.uniform_(-0.5, 0.5)
            m.out_proj.bias.uniform_(-0.5, 0.5)
        mods.append(m)
    memory = torch.randn(lk, b, e, device="cuda", requires_grad=True)
    mem_key = torch.randn(lk, b, e, device="cuda", requires_grad=True)
    queries = [torch.randn(lq, b, e, device="cuda") for _ in range(nl)]
    weights = [torch.randn(lq, b, e, device="cuda") for _ in range(nl)]
    used = [i != unused for i in range(nl)]
    params = [t for m in mods for t in (m.in_proj_weight, m.in_proj_bias, m.out_proj.weight, m.out_proj.bias)]

    # dropout: a pinned seed counter and known per-call salts, so that the reference can rebuild each layer's mask
    salts = [1000 + 17 * i for i in range(nl)]
    salt_iter = iter(salts)
    monkeypatch.setattr(attention_launch, "next_salt", lambda: next(salt_iter))
    attention_launch.seed_counter(memory.device).fill_(2024)

    bank, token = ops.kv_bank(mem_key, memory, mods)
    outs = [mods[i].forward_bank(queries[i], bank, token, i)[0] for i in range(nl)]
    loss = sum((outs[i] * weights[i]).sum() for i in range(nl) if used[i])
    _poison_free_blocks((lk * b, nl * e))
    grads = torch.autograd.grad(loss, [memory, mem_key, *params], allow_unused=True)

    mem64, key64 = (t.detach().double().requires_grad_(True) for t in (memory, mem_key))
    params64 = [t.detach().double().requires_grad_(True) for t in params]
    outs64 = []
    for i in range(nl):
        w, bias, wo, bo = params64[4 * i: 4 * i + 4]
        q = queries[i].double() @ w[:e].t() + bias[:e]
        k = key64 @ w[e: 2 * e].t() + bias[e: 2 * e]
        v = mem64 @ w[2 * e:].t() + bias[2 * e:]
        keep = attention_launch.dropout_keep(b * h, lq, lk, p, salts[i], memory.device) if p > 0 else None
        att = attention_sm100._math(q, k, v, h, p, True, False, keep)
        outs64.append(att @ wo.t() + bo)
    loss64 = sum((outs64[i] * weights[i].double()).sum() for i in range(nl) if used[i])
    ref = torch.autograd.grad(loss64, [mem64, key64, *params64], allow_unused=True)
    ref = [torch.zeros_like(t) if g is None else g for t, g in zip([mem64, key64, *params64], ref)]

    for i in range(nl):
        assert _rel(outs[i], outs64[i].detach()) < 1e-4, f"layer {i} output"
    assert _rel(grads[0], ref[0]) < 2e-4, "d memory"
    assert _rel(grads[1], ref[1]) < 2e-4, "d memory key"
    for i in range(nl):
        dw, db, dwo, dbo = grads[2 + 4 * i: 6 + 4 * i]
        rw, rb, rwo, rbo = ref[2 + 4 * i: 6 + 4 * i]
        if not used[i]:
            for g in (dw, db, dwo, dbo):
                assert g is None or not bool(g.any()), f"layer {i} is unused but has a non-zero gradient"
            continue
        for j, name in enumerate("qkv"):
            rows = slice(j * e, (j + 1) * e)
            assert _rel(dw[rows], rw[rows]) < 2e-4, f"layer {i} d in_proj_weight ({name})"
            # the key bias does not change the softmax: its exact gradient is zero, measured on the whole bias' scale
            assert _rel(db[rows], rb[rows], rb.abs().max()) < 2e-4, f"layer {i} d in_proj_bias ({name})"
        assert _rel(dwo, rwo) < 2e-4, f"layer {i} d out_proj.weight"
        assert _rel(dbo, rbo) < 2e-4, f"layer {i} d out_proj.bias"
