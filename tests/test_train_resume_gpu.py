"""TrainStep(optimizer=AdamW): checkpoints carry the optimizer state, and a resumed run is the run that never stopped.

  * exact resume: K captured steps, a checkpoint written the way the reference's save_checkpoint writes it, a fresh
    model / AdamW / TrainStep that loads it (before prepare, or after capture through the load_state_dict hook), K
    more steps == 2K steps without a break, bit for bit (parameters, both moments, step count);
  * interchange: a checkpoint of the plain eager loop (torch AdamW) is adopted bit for bit and continued within the
    eager-vs-graph bars, and TrainStep's checkpoint loads into a stock AdamW that continues the same way;
  * stage 1 -> stage 2: a stage-1 checkpoint continues under the stage-2 configuration (discovery on);
  * two ranks: rank 0's optimizer state wins at prepare (skipped on a single-GPU box)."""
import os
import socket
import tempfile
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

K = 3
_STAGE2 = dict(if_clip_weak_labels=True, loss_feat_seen_softmax_weakly_loss_with_novel_cate_confi_weight=1.0,
               confidence_type="clip-max-prob",
               online_nms_update_save_novel_label_clip_driven_with_cate_confidence=True, save_objectness=0.3,
               clip_driven_keep_thres=0.0258, online_nms_update_save_epoch=10)


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _args(**kw):
    from coda_neurips2023_b200 import synthetic

    # the region-embedding L1 loss off: its head then receives no gradient, and its parameters are inactive
    base = dict(nqueries=128, preenc_npoints=256, dec_dim=128, dec_nlayers=2, dec_ffn_dim=64, enc_dropout=0.0,
                dec_dropout=0.0, mlp_dropout=0.0, loss_predicted_region_embed_l1_weight=0.0, filter_biases_wd=True)
    return synthetic.make_args(**dict(base, **kw))


def _make(args, seed=0, device="cuda"):
    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.models import build_model

    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    return model.to(device).train(), build_criterion(args, cfg).to(device)


def _adamw(args, model):
    """the reference's build_optimizer (optimizer.py:5-36)"""
    from coda_neurips2023_b200.engine import _no_decay

    decay, no_decay = [], []
    for name, p in model.named_parameters():
        if p.requires_grad:
            (no_decay if args.filter_biases_wd and _no_decay(name, p) else decay).append(p)
    groups = ([{"params": no_decay, "weight_decay": 0.0}] if args.filter_biases_wd else []) + \
        [{"params": decay, "weight_decay": args.weight_decay}]
    return torch.optim.AdamW(groups, lr=args.base_lr)


def _batches(n):
    from coda_neurips2023_b200 import synthetic

    return [synthetic.to_device(synthetic.make_batch(2, 3000, seed=40 + i), "cuda") for i in range(n)]


def _epoch(i):
    return 2.0 * i      # the learning rate moves from step to step (warm-up)


def _run(step, batches, steps):
    for i in steps:
        np.random.seed(100 + i)          # the CLIP-crop box draw
        step(batches[i], _epoch(i))
    torch.cuda.synchronize()


def _save(path, model, opt, epoch=0):
    """what the reference's save_checkpoint writes"""
    torch.save({"model": model.state_dict(), "optimizer": opt.state_dict(), "epoch": epoch, "args": None,
                "best_val_metrics": {}}, path)


def _resume(path, model, opt):
    """what the reference's resume_if_possible loads"""
    sd = torch.load(path, map_location=torch.device("cpu"), weights_only=False)
    model.load_state_dict(sd["model"], strict=True)
    opt.load_state_dict(sd["optimizer"])
    return sd


def _bits(t):
    return t.detach().reshape(-1).view(torch.int32)


def _flat_state(step):
    o = step.optimizer
    return [step.flat.flat_param.detach().clone(), o.exp_avg.clone(), o.exp_avg_sq.clone(), float(o.state[0])]


@pytest.mark.parametrize("load", ["before_prepare", "after_capture"])
def test_resumed_run_is_bit_identical_to_the_unbroken_run(load, tmp_path):
    from coda_neurips2023_b200.engine import TrainStep

    args = _args()
    batches = _batches(2 * K)
    dev = torch.device("cuda", 0)
    model, crit = _make(args)
    opt = _adamw(args, model)
    step = TrainStep(args, model, crit, dev, optimizer=opt)
    np.random.seed(11)
    step.capture(batches[0], warmup=2)
    _run(step, batches, range(2 * K))
    want = _flat_state(step)
    want_sd = opt.state_dict()
    assert want[3] == 2 * K

    model1, crit1 = _make(args)
    opt1 = _adamw(args, model1)
    step1 = TrainStep(args, model1, crit1, dev, optimizer=opt1)
    np.random.seed(11)
    step1.capture(batches[0], warmup=2)
    _run(step1, batches, range(K))
    ckpt = str(tmp_path / "checkpoint.pth")
    _save(ckpt, model1, opt1, epoch=K)

    model2, crit2 = _make(args, seed=1)     # another initialisation: everything must come from the checkpoint
    opt2 = _adamw(args, model2)
    step2 = TrainStep(args, model2, crit2, dev, optimizer=opt2)
    if load == "before_prepare":
        _resume(ckpt, model2, opt2)
        np.random.seed(11)
        step2.capture(batches[0], warmup=2)
    else:
        np.random.seed(11)
        step2.capture(batches[0], warmup=2)
        graph = step2.graph
        _resume(ckpt, model2, opt2)          # the load_state_dict hook imports the state in place
        assert step2.graph is graph
    assert float(step2.optimizer.state[0]) == K
    _run(step2, batches, range(K, 2 * K))
    assert step2.flat.names == step.flat.names
    got = _flat_state(step2)
    for name, g, w in zip(("parameters", "exp_avg", "exp_avg_sq"), got[:3], want[:3]):
        assert torch.equal(_bits(g), _bits(w)), name
    assert got[3] == want[3]
    got_sd = opt2.state_dict()
    assert got_sd["param_groups"] == want_sd["param_groups"]
    assert sorted(got_sd["state"]) == sorted(want_sd["state"])
    for k, st in want_sd["state"].items():
        for key, t in st.items():
            assert torch.equal(_bits(got_sd["state"][k][key]), _bits(t)), (k, key)


def test_in_memory_reload_and_a_later_step_taking_the_optimizer_over():
    """opt.load_state_dict(opt.state_dict()) after capture (torch keeps the views of the flat buffers as they are)
    changes nothing: the run stays bit-identical to one without the reload.  A second TrainStep that adopts the same
    optimizer holds its hooks from then on: state_dict() reads, and load_state_dict() writes, the second step's
    buffers, and the first step's are left alone."""
    from coda_neurips2023_b200.engine import TrainStep

    args = _args()
    batches = _batches(2 * K)
    dev = torch.device("cuda", 0)
    model, crit = _make(args)
    step = TrainStep(args, model, crit, dev, optimizer=_adamw(args, model))
    np.random.seed(11)
    step.capture(batches[0], warmup=2)
    _run(step, batches, range(2 * K))
    want = _flat_state(step)

    model1, crit1 = _make(args)
    opt1 = _adamw(args, model1)
    step1 = TrainStep(args, model1, crit1, dev, optimizer=opt1)
    np.random.seed(11)
    step1.capture(batches[0], warmup=2)
    _run(step1, batches, range(K))
    opt1.load_state_dict(opt1.state_dict())
    assert float(step1.optimizer.state[0]) == K and step1.optimizer.exp_avg.abs().sum() > 0
    _run(step1, batches, range(K, 2 * K))
    got = _flat_state(step1)
    for name, g, w in zip(("parameters", "exp_avg", "exp_avg_sq"), got[:3], want[:3]):
        assert torch.equal(_bits(g), _bits(w)), name
    assert got[3] == want[3]

    step_b = TrainStep(args, model1, crit1, dev, optimizer=opt1)    # rebuilt over the same model and optimizer
    np.random.seed(11)
    step_b.prepare(batches[0])
    fb, f1 = step_b.optimizer, step1.optimizer
    assert float(fb.state[0]) == 2 * K
    assert step_b.flat.names == step1.flat.names
    assert torch.equal(fb.exp_avg, f1.exp_avg) and torch.equal(fb.exp_avg_sq, f1.exp_avg_sq)
    sd = opt1.state_dict()
    lo, hi = fb.exp_avg.data_ptr(), fb.exp_avg.data_ptr() + 4 * fb.exp_avg.numel()
    assert all(lo <= st["exp_avg"].data_ptr() < hi for st in sd["state"].values())
    m1 = f1.exp_avg.clone()
    doubled = {"param_groups": sd["param_groups"],
               "state": {k: {"step": st["step"].clone(), "exp_avg": st["exp_avg"].cpu() * 2,
                             "exp_avg_sq": st["exp_avg_sq"].cpu()} for k, st in sd["state"].items()}}
    opt1.load_state_dict(doubled)
    assert torch.equal(fb.exp_avg, m1 * 2)
    assert torch.equal(f1.exp_avg, m1), "the first step's hooks still import into its buffers"


def _eager_step(model, crit, opt, args, batch, i):
    """the reference's loop body (engine.py:120-165) with torch's AdamW"""
    from coda_neurips2023_b200.engine import adjust_learning_rate

    adjust_learning_rate(args, opt, 0.0)
    np.random.seed(100 + i)
    opt.zero_grad()
    out = model(batch, curr_epoch=0)
    loss, _ = crit(out, batch)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(model.parameters(), args.clip_gradient)
    opt.step()


def _assert_close_params(a, b):
    changed = 0
    pb = dict(b.named_parameters())
    for n, p in a.named_parameters():
        if p.requires_grad:
            assert torch.allclose(p, pb[n], rtol=1e-4, atol=1e-6), n
            changed += 1
    assert changed > 100


def test_torch_adamw_checkpoint_interchanges_with_the_flat_step(tmp_path):
    from coda_neurips2023_b200.engine import TrainStep, adamw_flat_index

    args = _args()
    batches = _batches(K + 5)
    dev = torch.device("cuda", 0)
    # the plain eager loop, K steps, then its checkpoint
    model_e, crit_e = _make(args)
    opt_e = _adamw(args, model_e)
    for i in range(K):
        _eager_step(model_e, crit_e, opt_e, args, batches[i], i)
    ckpt = str(tmp_path / "eager.pth")
    _save(ckpt, model_e, opt_e)
    # TrainStep adopts it
    model_t, crit_t = _make(args, seed=1)
    opt_t = _adamw(args, model_t)
    sd = _resume(ckpt, model_t, opt_t)["optimizer"]
    step = TrainStep(args, model_t, crit_t, dev, optimizer=opt_t)
    np.random.seed(11)
    step.capture(batches[0], warmup=2)
    index = adamw_flat_index(opt_t, step.flat)
    fa = step.optimizer
    assert float(fa.state[0]) == K
    nstate = 0
    for i, p in enumerate(step.flat.params):
        st = sd["state"].get(index[i])
        if st is None:
            continue
        off, n = step.flat.offsets[i], p.numel()
        assert torch.equal(_bits(fa.exp_avg[off:off + n].cpu()), _bits(st["exp_avg"])), step.flat.names[i]
        assert torch.equal(_bits(fa.exp_avg_sq[off:off + n].cpu()), _bits(st["exp_avg_sq"])), step.flat.names[i]
        nstate += 1
    assert nstate == sum(fa.active) and nstate == len(sd["state"])
    # 3 steps each way from the same state
    for i in range(K, K + 3):
        np.random.seed(100 + i)
        step(batches[i], 0.0)
        _eager_step(model_e, crit_e, opt_e, args, batches[i], i)
    torch.cuda.synchronize()
    _assert_close_params(model_t, model_e)
    # the reverse: TrainStep's checkpoint into a stock AdamW that continues
    ckpt_t = str(tmp_path / "flat.pth")
    _save(ckpt_t, model_t, opt_t)
    model_r, crit_r = _make(args, seed=2)
    opt_r = _adamw(args, model_r)
    sd_t = _resume(ckpt_t, model_r, opt_r)["optimizer"]
    assert all(float(st["step"]) == K + 3 for st in sd_t["state"].values())
    for k, st in opt_r.state_dict()["state"].items():
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(_bits(st[key].cpu()), _bits(sd_t["state"][k][key])), (k, key)
    for i in range(K + 3, K + 5):
        np.random.seed(100 + i)
        step(batches[i], 0.0)
        _eager_step(model_r, crit_r, opt_r, args, batches[i], i)
    torch.cuda.synchronize()
    _assert_close_params(model_t, model_r)


def test_stage1_checkpoint_continues_in_stage2(tmp_path):
    from coda_neurips2023_b200.engine import TrainStep

    dev = torch.device("cuda", 0)
    # the scripts' region-embedding L1 weight: stage 2's weak-label loss trains that head, so stage 1 must too (a
    # stage-1 run without it leaves the head with no AdamW state, which the flat step's single step count refuses)
    args1 = _args(loss_predicted_region_embed_l1_weight=1.0)
    batches = _batches(K + 1)
    model1, crit1 = _make(args1)
    opt1 = _adamw(args1, model1)
    step1 = TrainStep(args1, model1, crit1, dev, optimizer=opt1)
    np.random.seed(11)
    step1.capture(batches[0], warmup=2)
    _run(step1, batches, range(K))
    ckpt = str(tmp_path / "last_checkpoint.pth")
    _save(ckpt, model1, opt1, epoch=K)
    m_ckpt = step1.optimizer.exp_avg.clone()
    v_ckpt = step1.optimizer.exp_avg_sq.clone()

    args2 = _args(checkpoint_file=ckpt, loss_predicted_region_embed_l1_weight=1.0, **_STAGE2)
    model2, crit2 = _make(args2, seed=1)
    opt2 = _adamw(args2, model2)
    _resume(args2.checkpoint_file, model2, opt2)
    step2 = TrainStep(args2, model2, crit2, dev, optimizer=opt2)
    batch = dict(batches[K])
    pseudo = tempfile.mkdtemp(prefix="coda_resume_pseudo_", dir=tmp_path)
    batch["pseudo_box_path"] = [os.path.join(pseudo, f"scene{i}.npy") for i in range(2)]
    np.random.seed(11)
    step2.capture(batch, warmup=1)
    assert step2._branch(0.0)[2], "discovery is not on in the stage-2 configuration"
    assert step2.flat.names == step1.flat.names
    np.random.seed(100 + K)
    step2(batch, 0.0)
    torch.cuda.synchronize()
    fa = step2.optimizer
    assert float(fa.state[0]) == K + 1
    # m <- b1 m + (1 - b1) c g, v <- b2 v + (1 - b2) (c g)^2 with the clip coefficient c of this step, active ranges
    b1, b2 = fa.betas
    g = step2.flat.flat_grad * fa.state[2]
    live = torch.zeros_like(g, dtype=torch.bool)
    for i, p in enumerate(step2.flat.params):
        if fa.active[i]:
            live[step2.flat.offsets[i]:step2.flat.offsets[i] + p.numel()] = True
    # (the kernel takes beta and 1 - beta in fp32; the two terms cancel in m: the bar is on their magnitudes)
    for got, old, new, b in ((fa.exp_avg, m_ckpt, g, b1), (fa.exp_avg_sq, v_ckpt, g * g, b2)):
        b = torch.tensor(b, dtype=torch.float32, device=g.device)
        exp = torch.where(live, b * old + (1 - b) * new, old)
        # floor: fp32 denormals (v of an element whose gradient is ~1e-20), which the kernel may flush
        bar = 1e-6 * torch.where(live, (b * old).abs() + ((1 - b) * new).abs(), 0.0) + 1e-37
        assert ((got - exp).abs() <= bar).all(), float(((got - exp).abs() - bar).max())
    assert not torch.equal(fa.exp_avg, m_ckpt)
    assert all(float(st["step"]) == K + 1 for st in opt2.state_dict()["state"].values())


# ------------------------------------------------------------------ two ranks
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.engine import TrainStep

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    args = _args(ngpus=2)
    model, crit = _make(args, seed=100 + rank, device=dev)
    opt = _adamw(args, model)
    g = torch.Generator(device=dev).manual_seed(7 + rank)     # a different optimizer state on each rank
    for grp in opt.param_groups:
        for p in grp["params"]:
            opt.state[p] = {"step": torch.tensor(float(5 + 10 * rank)),
                            "exp_avg": torch.randn(p.shape, device=dev, generator=g) * 1e-3,
                            "exp_avg_sq": torch.rand(p.shape, device=dev, generator=g) * 1e-6}
    batch = synthetic.to_device(synthetic.make_batch(2, 3000, seed=7 + rank), dev)
    step = TrainStep(args, model, crit, dev, optimizer=opt)
    np.random.seed(3)
    step.prepare(batch)
    fa = step.optimizer
    spread = 0.0
    for t in (fa.exp_avg, fa.exp_avg_sq, fa.state[:1]):
        hi, lo = t.clone(), t.clone()
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        spread = max(spread, float((hi - lo).abs().max()))
    sd = opt.state_dict()
    ret[f"steps{rank}"] = sorted({float(st["step"]) for st in sd["state"].values()})
    ret[f"nstate{rank}"] = len(sd["state"])
    if rank == 0:
        ret["spread"] = spread
    dist.barrier()
    os._exit(0)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_take_rank0_optimizer_state(built_lib):
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    assert ret["spread"] == 0.0, "rank 0's optimizer state was not broadcast"
    assert ret["steps0"] == ret["steps1"] == [5.0]
    assert ret["nstate0"] == ret["nstate1"]
