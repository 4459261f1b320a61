"""--if_clip_superset on the H100: the contrastive-loss row kernels coda_text_ce_fwd / _bwd against an fp64 restatement
(shapes, label / weight / embedding edges, guard words, repeatability), the whole superset loss (wgmma GEMM + row
kernels) against the ATen path, the two stage-2 superset cases against the reference's goldens, the captured step
against the eager one, and the pseudo-label class ids against the superset."""
import ctypes
import tempfile
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import model_parity_common as mpc
import superset_common as ssc
from coda_neurips2023_b200 import ops, synthetic
from coda_neurips2023_b200._lib import lib

pytestmark = pytest.mark.gpu

GUARD = 4          # guard floats on each side of every output (16 bytes: keeps the outputs 16-byte aligned)
SENTINEL = 12345.678


@pytest.fixture(autouse=True)
def _lib(built_lib):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _guarded(n, dev):
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.float32, device=dev)
    return buf, buf[GUARD:GUARD + n]


def _guards_intact(buf):
    return bool((buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all())


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _kernels(S, e, label, w, scale, g, c):
    """one forward + backward through the C entry points, every output between guard words"""
    rows, ld = S.shape
    d = e.shape[1]
    dev = S.device
    bufs = [_guarded(rows, dev) for _ in range(3)] + [_guarded(rows * ld, dev), _guarded(rows * d, dev)]
    (lb, loss), (sb, lse), (ib, inv), (db, ds), (nb, dn) = bufs
    st = torch.cuda.current_stream().cuda_stream
    L, ll, i = lib(), ctypes.c_longlong, ctypes.c_int
    assert L.coda_text_ce_fwd(ll(rows), i(c), i(ld), i(d), _p(S), _p(e), _p(label), _p(w), _p(scale), _p(loss),
                              _p(lse), _p(inv), ctypes.c_void_p(st)) == 0
    assert L.coda_text_ce_bwd(ll(rows), i(c), i(ld), i(d), _p(S), _p(e), _p(label), _p(w), _p(scale), _p(lse),
                              _p(inv), _p(g), _p(ds), _p(dn), ctypes.c_void_p(st)) == 0
    torch.cuda.synchronize()
    assert all(_guards_intact(b) for b, _ in bufs)
    return loss.clone(), ds.view(rows, ld).clone(), dn.view(rows, d).clone()


def _ref64(S, e, label, w, scale, g, c):
    """fp64 restatement of include/coda_step.h: per-row loss, dS (rows, ld), the normalisation term (rows, d)"""
    S, e, w, g = (t.double().cpu() for t in (S, e, w, g))
    label = label.cpu()
    s = float(scale)
    n = e.norm(dim=1)
    inv = 1.0 / (n + 1e-32)
    z = s * inv[:, None] * S[:, :c]
    lse = torch.logsumexp(z, dim=1)
    ok = (label >= 0) & (label < c)
    y = label.clamp(0, c - 1)
    loss = w * (lse - z.gather(1, y[:, None])[:, 0])
    loss = torch.where(label == -100, torch.zeros_like(loss), torch.where(ok, loss, torch.full_like(loss, np.nan)))
    G = (g * w)[:, None] * (torch.softmax(z, dim=1) - F.one_hot(y, c).double())
    G = torch.where(ok[:, None], G, torch.zeros_like(G))
    ds = torch.zeros_like(S)
    ds[:, :c] = s * inv[:, None] * G
    coef = torch.where(n > 0, -(inv / torch.where(n > 0, n, torch.ones_like(n))) * (G * z).sum(dim=1), torch.zeros_like(n))
    return loss, ds, coef[:, None] * e


def _case(rows, c, d=512, s=100.0, seed=0, dev="cuda"):
    g = torch.Generator().manual_seed(seed * 7919 + rows * 31 + c)
    ld = (c + 3) // 4 * 4
    t = torch.randn(c, d, generator=g)
    t = t / t.norm(dim=1, keepdim=True)
    e = torch.randn(rows, d, generator=g)
    label = torch.randint(0, c, (rows,), generator=g)
    w = torch.rand(rows, generator=g)
    if rows >= 8:
        w[1] = 0.0                       # weight 0
        label[2] = c - 1                 # last class
        label[3] = -100                  # ignore_index
        e[4] = 0.0                       # zero embedding
        if c >= 4:
            # text rows 0..3 nearly parallel, and rows 5..7 nearly parallel to text row 0: at s = 100 their logits
            # are close to 100 and close to each other, so the softmax splits between them
            for j in range(1, 4):
                t[j] = t[0] + 0.01 * torch.randn(d, generator=g)
            t = t / t.norm(dim=1, keepdim=True)
            for r in range(5, 8):
                e[r] = 3.0 * t[0] + 3e-3 * torch.randn(d, generator=g)
                label[r] = r - 5
    S = torch.zeros(rows, ld)
    S[:, :c] = e.double().mm(t.double().t()).float()
    S[:, c:] = 777.0                     # padding columns: never read as logits
    gout = torch.rand(rows, generator=g) + 0.5
    return (S.to(dev), e.to(dev), label.to(dev), w.to(dev), torch.tensor([s], device=dev), gout.to(dev))


def _check(got, ref, args, c):
    """loss within 5e-5 * max(1, |ref|); dS and the normalisation term within 2e-5 of the row's max |ref| plus what
    the fp32 rounding of the logits allows: a logit z near 100 is rounded by up to ~1e-5, which moves the softmax
    by ~1e-5 * p and so dS by up to 1e-5 * scale * inv * |g w|, the normalisation term by 1e-5 * inv * |g w| (its
    entries are coef * e with |e_k| <= ||e||).  That allowance matters only in rows whose gradient is small (a
    confident, correct row), where no fp32 evaluation of the logits can meet a relative bar."""
    loss, ds, dn = got
    rl, rds, rdn = ref
    _, e, _, w, scale, g = args
    loss, ds, dn = loss.double().cpu(), ds.double().cpu(), dn.double().cpu()
    fin = torch.isfinite(rl)
    assert torch.equal(torch.isnan(loss), ~fin)
    assert ((loss[fin] - rl[fin]).abs() <= 5e-5 * rl[fin].abs().clamp(min=1.0)).all(), \
        float(((loss[fin] - rl[fin]).abs() / rl[fin].abs().clamp(min=1.0)).max())
    inv = 1.0 / (e.double().cpu().norm(dim=1) + 1e-32)
    gw = (g.double() * w.double()).abs().cpu()
    for got_, ref_, slack in ((ds, rds, 1e-5 * float(scale) * inv * gw), (dn, rdn, 1e-5 * inv * gw)):
        got_, ref_ = got_[fin], ref_[fin]
        bar = 2e-5 * ref_.abs().max(dim=1, keepdim=True).values + slack[fin][:, None]
        assert ((got_ - ref_).abs() <= bar).all(), float(((got_ - ref_).abs() - bar).max())
    assert (ds[:, c:] == 0).all()


@pytest.mark.parametrize("c", [1, 10, 232, 1201, 1203])
@pytest.mark.parametrize("rows", [1, 63, 64, 65, 1024, 7168, 8192])
def test_text_ce_kernels_match_fp64(rows, c):
    args = _case(rows, c)
    got = _kernels(*args, c)
    _check(got, _ref64(*args, c), args, c)
    again = _kernels(*args, c)
    for a, b in zip(got, again):       # the same bits on every run
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("bad", [1201, 5000, -1])
def test_out_of_range_label_gives_a_nan_row_and_nothing_else(bad):
    S, e, label, w, scale, g = _case(64, 1201)
    label[7] = bad
    got = _kernels(S, e, label, w, scale, g, 1201)
    loss, ds, dn = got
    assert torch.isnan(loss[7]) and torch.isnan(ds[7, :1201]).all() and torch.isnan(dn[7]).all()
    keep = torch.ones(64, dtype=torch.bool)
    keep[7] = False
    args = (S, e, label, w, scale, g)
    _check(tuple(t[keep.cuda()] for t in got), tuple(t[keep] for t in _ref64(*args, 1201)),
           tuple(t if t.numel() == 1 else t[keep.cuda()] for t in args), 1201)


def test_superset_loss_matches_the_aten_path():
    """GEMM + row kernels against the ATen path (normalise, fp32 matmul, scale, cross-entropy) at R = 8192 rows
    (8 scenes x 128 queries x 8 decoder layers) and C = 1201."""
    rows, c, d = 8192, 1201, 512
    g = torch.Generator().manual_seed(3)
    t = torch.randn(c, d, generator=g)
    t = (t / t.norm(dim=1, keepdim=True)).cuda()
    e0 = torch.randn(rows, d, generator=g).cuda()
    label = torch.randint(0, c, (rows,), generator=g).cuda()
    w = (torch.rand(rows, generator=g) > 0.3).float().cuda()
    scale = torch.tensor([100.0], device="cuda")
    e = e0.clone().requires_grad_(True)
    loss = ops.text_contrastive_ce(e, t, label, w, scale).sum()
    loss.backward()
    er = e0.clone().requires_grad_(True)
    en = er / (er.norm(dim=-1, keepdim=True) + 1e-32)
    ref = (F.cross_entropy(en.mm(t.t()) * scale, label, reduction="none") * w).sum()
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)), (float(loss), float(ref))
    err = float((e.grad - er.grad).abs().max() / er.grad.abs().max())
    assert err <= 1e-4, err


@pytest.mark.parametrize("name", list(ssc.CASES))
def test_superset_step_matches_reference_golden(name):
    """Bars of the existing goldens on the H100: 1e-4 relative on outputs and losses, 5e-3 on gradients."""
    torch.manual_seed(0)
    model, out, loss, loss_dict, golden = ssc.run(name, "cuda")
    ssc.check_text_features(model, golden, rtol=1e-4)
    errs = mpc.compare(model, out, loss, loss_dict, golden, rtol=1e-4, atol=1e-5, grad_rtol=5e-3)
    worst = max(errs, key=errs.get)
    print(f"{name}: worst {worst} = {errs[worst]:.2e}")


def test_superset_pseudo_label_classes_index_the_superset():
    """flush_pseudo_labels writes class ids of superset rows: novel ones (>= train_range_max), < len(superset)."""
    model, out, loss, loss_dict, golden = ssc.run("stage2_superset", "cuda")
    paths = model._pending_pseudo["paths"]
    saved = model.flush_pseudo_labels()
    ids = np.concatenate([a[:, 7] for a in saved])
    assert ids.size > 0 and np.array_equal(ids, golden["pseudo.rows"][:, 7])
    assert (ids == np.round(ids)).all() and (ids >= model.train_range_max).all()
    assert (ids < len(model.superset_all_classes_keys)).all()
    on_disk = np.concatenate([np.load(p)[:, 7] for p, a in zip(paths, saved) if len(a)])
    assert np.array_equal(on_disk, ids)


def test_captured_superset_step_equals_the_eager_step(tmp_path, monkeypatch):
    """Stage 2 with the superset (1201 seeded text rows: no class lists here), weak labels and discovery on, 8 scenes
    x 20 000 points, 128 queries: the first replay of TrainStep's CUDA graph gives the eager step's loss."""
    from coda_neurips2023_b200 import attention_launch
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.engine import TrainStep
    from coda_neurips2023_b200.models import build_model

    monkeypatch.chdir(tmp_path)
    args = synthetic.make_args(
        dataset_name="sunrgbd_anonymous_aligned_image_with_novel_cate_confi", nqueries=128, train_range_max=10,
        test_range_max=46, if_clip_superset=True, if_clip_weak_labels=True,
        loss_feat_seen_softmax_weakly_loss_with_novel_cate_confi_weight=1.0, confidence_type="non-confidence",
        online_nms_update_save_novel_label_clip_driven_with_cate_confidence=True, save_objectness=0.3,
        clip_driven_keep_thres=0.3, online_nms_update_save_epoch=50, distillation_box_num=32,
        enc_dropout=0.0, dec_dropout=0.0, mlp_dropout=0.0)
    cfg = synthetic.SyntheticDatasetConfig(args)

    def make():
        torch.manual_seed(0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = build_model(args, cfg)
        return model.cuda().train(), build_criterion(args, cfg).cuda()

    tmp = tempfile.mkdtemp(prefix="coda_superset_pseudo_")
    batches = []
    for s in range(2):
        bt = synthetic.to_device(synthetic.make_batch(8, 20000, seed=30 + s), "cuda")
        bt["pseudo_box_path"] = [f"{tmp}/s{s}_scene{i}.npy" for i in range(8)]
        batches.append(bt)
    model, crit = make()
    assert model.superset_text_features_fg_norm.shape == (1201, 512)
    seed0 = int(attention_launch.seed_counter(torch.device("cuda", 0)))
    step = TrainStep(args, model, crit, torch.device("cuda", 0))
    np.random.seed(11)
    step.capture(batches[0], warmup=2)
    losses = []
    for i, bt in enumerate(batches):
        np.random.seed(12 + i)
        losses.append(float(step(bt, 0.0)[0]))
    assert all(np.isfinite(losses)), losses
    model2, crit2 = make()
    attention_launch.seed_counter(torch.device("cuda", 0)).fill_(seed0)
    step2 = TrainStep(args, model2, crit2, torch.device("cuda", 0))
    step2.prepare(batches[0])
    np.random.seed(12)
    loss_e = float(step2(batches[0], 0.0)[0])
    print(f"superset stage-2 step: graph losses {losses}, eager {loss_e}")
    assert abs(loss_e - losses[0]) <= 1e-5 * abs(losses[0])
