"""Models converted by torch.nn.SyncBatchNorm.convert_sync_batchnorm, as the reference's main.py does before it trains
or tests on more than one GPU (main.py:992-996), run on this package's kernels.

1. One process, no process group: a converted model gives the unconverted model's bits (loss, every gradient, every
   running statistic; eval-mode outputs of the CoDA head and of the baseline head), and its eval-mode pre-encoder
   runs on the fused inference kernel.
2. Three gloo ranks sharing cuda:0, the converted model wrapped in DistributedDataParallel(find_unused_parameters=
   False) and run through the reference's own training loop (engine.py:130-164: zero_grad, forward through DDP,
   criterion, backward, clip_grad_norm_, AdamW step) for three steps:
     (a) right after DDP is constructed, every rank's forward on one shared input gives rank 0's bits: DDP's
         broadcast moved every rank's parameters, so no weight planes packed before it may be used;
     (b) the first step's all-reduced gradients and running statistics equal those of TrainStep(sync_bn=True) on the
         unconverted model, on the same ranks and batches;
     (c) the same first-step gradients and running statistics equal those of ONE process on the concatenated batch
         with the unconverted model (plain per-GPU BatchNorm kernels over all the rows), within the reorder-noise
         yardstick of tests/test_nccl_gpu.py;
     (d) DDP raises no unused-parameter error, and the parameters are bit-identical across ranks after every step.
   The ranks start from different parameters and buffers (rank r adds r * 1e-3), so that the broadcast matters.
3. engine.evaluate on the converted, DDP-wrapped model on the same gloo ranks, each fed its DistributedSampler share,
   gives the metrics of engine.evaluate in one process with the unconverted model over the stream the ranks'
   all-gather builds."""
import datetime
import os
import socket
import tempfile
import warnings

import numpy as np
import pytest
import torch

import baseline_eval_common as bec
import test_eval_distributed_gpu as ED
import model_parity_common as mpc
import scannet_parity_common as spc
from running_stats_fill import fill_running_stats_by_name

pytestmark = pytest.mark.gpu

WORLD = 3
SCENES_PER_RANK = 2
BASELINE = "baseline_stage1_small"
BASELINE_ARGS = dict(mpc._SMALL, model_name="3detrmulticlasshead", loss_predicted_region_embed_l1_weight=0.0)
DDP_CASES = ("stage1_small", "stage2_discovery", "masked_small", BASELINE, "scannet_stage1_small")
STEPS = 3
# (b): the DDP run and the TrainStep run execute the same kernels on the same rows; they differ in how the three
# ranks' gradients are summed (DDP divides each rank's gradient by 3 before its all-reduce, TrainStep divides the
# sum).  The deviation is held against the largest gradient entry of the whole model: with synchronised BatchNorm a
# per-channel constant in front of a Linear + BatchNorm (encoder.layers.2.linear2.bias, ahead of the encoder-to-decoder
# projection) has a rank-summed gradient that is zero in exact arithmetic, while each rank's own gradient is not, so
# relative to its own tensor the reordered sum of three cancelling terms differs by several per cent (measured 3.4e-2
# .. 7.3e-2 on an H100 80GB HBM3), which says nothing about the exchange.  Against the largest gradient the five
# cases measured 7.3e-8 .. 3.4e-7 there (H100 80GB HBM3, 700 W).
GRAD_BAR = 1e-6          # max |difference| / max |TrainStep gradient| over every parameter
# Every tensor whose gradient is not pure rounding is held to its own largest entry as well.  Pure rounding is
# measured, not listed: the tensors whose single-process gradient moves by more than ROUNDING_NOISE (relative L2) when
# the same scenes are visited in another order (CONCAT_PERMS below).  Measured on an H100 80GB HBM3 (700 W) these are
# the biases in front of a Linear + BatchNorm -- encoder.layers.2.linear2.bias, decoder.norm.bias and, in the masked
# encoder, encoder.layers.0.linear2.bias (reorder noise 1.0 .. 1.2; against their own largest entry the DDP / TrainStep
# difference is 1.2e-2 .. 2.1e-2) -- and they are held to GRAD_BAR only.  Every other tensor measured at most 1.7e-6
# of its own largest entry.
OWN_BAR = 1e-5
ROUNDING_NOISE = 0.1
# (c): rank-summed gradients against one process on the concatenated batch.  Both compute the same mathematics but
# reduce in another order everywhere, and training-mode BatchNorm amplifies the rounding of the two-plane gradient
# GEMMs, so each parameter is held to a few times ITS OWN reorder noise: the same single process with the scenes in
# three other orders (tests/test_nccl_gpu.py, test_two_rank_sync_batchnorm_equals_concatenated_batch).
CONCAT_NOISE_FACTOR, CONCAT_FLOOR = 6.0, 3e-3
CONCAT_STATS_BAR = 1e-4  # running mean / var, max |difference| / max |value|
CONCAT_PERMS = ((0, 1, 2, 3, 4, 5), (2, 3, 4, 5, 0, 1), (1, 0, 3, 2, 5, 4), (5, 4, 3, 2, 1, 0))
# stage-2's weak-label loss divides by the LOCAL count of confident queries (reference criterion.py:598-645), so the
# mean over ranks is not the loss of the concatenated batch: that case is left out of (c) only
CONCAT_CASES = tuple(n for n in DDP_CASES if n != "stage2_discovery")
STATS_BAR = 0.0          # running statistics: the same collectives on the same sums, bit for bit


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _convert(model):
    model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    assert any(isinstance(m, torch.nn.SyncBatchNorm) for m in model.modules())
    return model


# --------------------------------------------------------------------------- 1. one process, no process group
def _train_step_bits(convert):
    args, model, crit, inputs, _ = mpc.build("stage1_small", "cuda")
    if convert:
        model = _convert(model)
    np.random.seed(123)
    out = model(inputs, curr_epoch=0)
    loss, _ = crit(out, inputs)
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.requires_grad}
    bufs = {n: b.detach().clone() for n, b in model.named_buffers()}
    return loss.detach().clone(), grads, bufs


def _same_bits(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert torch.equal(a[k], b[k]), f"{what} {k}"


def test_converted_model_trains_with_the_unconverted_bits():
    assert not torch.distributed.is_initialized()
    loss0, g0, b0 = _train_step_bits(False)
    loss1, g1, b1 = _train_step_bits(True)
    assert torch.equal(loss0, loss1)
    _same_bits(g0, g1, "gradient")
    _same_bits(b0, b1, "buffer")
    print(f"PARITY sync_bn_modules one process, stage1_small: loss, {len(g0)} gradients and {len(b0)} buffers "
          "bit-identical (bar: 0)")


def _spy_infer(monkeypatch):
    from coda_neurips2023_b200 import sa_mlp

    calls = []
    real = sa_mlp.shared_mlp_max_infer

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(sa_mlp, "shared_mlp_max_infer", spy)
    return calls


def _coda_eval(convert):
    _, model, _, inputs, _ = mpc.build("stage1_small", "cuda")
    fill_running_stats_by_name(model, seed=7)
    if convert:
        model = _convert(model)
    model.eval()
    with torch.no_grad():
        out = model(inputs, if_real_test=True)["outputs"]
    return {k: v for k, v in out.items() if isinstance(v, torch.Tensor)}


def _baseline_eval(convert):
    with bec.class_lists():
        model, _ = bec.build_ours("cuda")
        if convert:
            model = _convert(model).eval()
        with torch.no_grad():
            out = model(bec.test_batch("cuda"), if_real_test=True)["outputs"]
    return {k: v for k, v in out.items() if isinstance(v, torch.Tensor)}


@pytest.mark.parametrize("head", ["coda", "baseline"])
def test_converted_model_evaluates_with_the_unconverted_bits_on_the_fused_kernel(head, monkeypatch):
    run = _coda_eval if head == "coda" else _baseline_eval
    plain = run(False)
    calls = _spy_infer(monkeypatch)
    converted = run(True)
    assert calls, "the converted model's pre-encoder did not run the fused inference kernel"
    _same_bits(plain, converted, f"{head} output")
    print(f"PARITY sync_bn_modules eval {head}: {len(plain)} outputs bit-identical (bar: 0), fused kernel calls "
          f"{len(calls)}")


# --------------------------------------------------------------------------- 2. gloo ranks, DDP
def _build(name, dev):
    """OUR model and criterion for a case, in training mode on `dev`, and the case's full batch (WORLD ranks' scenes)."""
    if name == BASELINE:
        from coda_neurips2023_b200 import synthetic
        from coda_neurips2023_b200.criterion import build_criterion
        from coda_neurips2023_b200.models import build_model
        from param_fill import fill_by_name

        args = synthetic.make_args(**BASELINE_ARGS)
        cfg = synthetic.SyntheticDatasetConfig(args)
        torch.manual_seed(0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = build_model(args, cfg)
        fill_by_name(model, seed=3)
        model.to_device(dev)
        crit = build_criterion(args, cfg).to(dev)
        extra = {}
        batch = synthetic.make_batch(WORLD * SCENES_PER_RANK, 3000, seed=5)
    elif name in spc.CASES:
        from coda_neurips2023_b200 import synthetic

        args, model, crit, _, _ = spc.build(name, dev)
        extra = spc.CASES[name][3]
        batch = synthetic.make_batch(WORLD * SCENES_PER_RANK, spc.CASES[name][1], seed=5, image_hw=spc.IMAGE_HW,
                                     camera="scannet")
    else:
        from coda_neurips2023_b200 import synthetic

        args, model, crit, _, _ = mpc.build(name, dev)
        _, npoints, _, extra = mpc.case(name)
        batch = synthetic.make_batch(WORLD * SCENES_PER_RANK, npoints, seed=5,
                                     image_hw=extra.get("image_hw", (531, 730)))
    model.train()
    if getattr(model, "clip_model", None) is not None:
        model.clip_model.eval()
    _normalise_region_embed_globally(crit)
    return args, model, crit, batch, extra


def _normalise_region_embed_globally(crit):
    """The cross-modal alignment loss divides by the LOCAL number of valid crops (reference criterion.py:924-943), so
    the mean of the ranks' losses is not the loss of the concatenated batch.  Every run of this module (DDP, TrainStep
    and the single process) rescales it by local / rank-averaged count instead, which makes it the concatenated
    batch's; with one process the factor is 1.  Dropping the loss instead is not possible: the text-correlation head
    would get no gradient, and DDP(find_unused_parameters=False) would raise, as it would for the reference."""
    from coda_neurips2023_b200.utils.dist import all_reduce_average

    key = "loss_predicted_region_embed_l1"
    local = crit.loss_functions[key]

    def rescaled(outputs, targets, assignments):
        out = local(outputs, targets, assignments)
        w = targets["gt_text_correlation_embedding_mask"].sum().float()
        out[key] = out[key] * (w / all_reduce_average(w))
        return out

    crit.loss_functions[key] = rescaled


def _rank_inputs(name, rank, dev, batch, extra, tmp):
    from coda_neurips2023_b200 import synthetic

    os.makedirs(tmp, exist_ok=True)
    sl = slice(rank * SCENES_PER_RANK, (rank + 1) * SCENES_PER_RANK)
    inputs = synthetic.to_device({k: v[sl] for k, v in batch.items()}, dev)
    if extra.get("pseudo"):
        inputs["pseudo_box_path"] = [os.path.join(tmp, f"{name}_r{rank}_s{i}.npy") for i in range(SCENES_PER_RANK)]
    return inputs


def _perturb(model, rank):
    """rank r's parameters and floating buffers + r * 1e-3: what DDP's broadcast has to undo"""
    with torch.no_grad():
        for t in list(model.parameters()) + list(model.buffers()):
            if t.dtype.is_floating_point:
                t.add_(rank * 1e-3)


def _fix_selection(model, rank):
    sel = np.random.RandomState(5).choice(128, size=(WORLD * SCENES_PER_RANK, 32))
    model.draw_box_selection = lambda bsz: sel[rank * SCENES_PER_RANK:(rank + 1) * SCENES_PER_RANK].astype(np.int64)


def _spread(t):
    import torch.distributed as dist

    hi, lo = t.clone(), t.clone()
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    return float((hi - lo).abs().max())


def _flat(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])


def _ddp_case(name, rank, dev, tmp):
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP

    from coda_neurips2023_b200 import ops

    res = {}
    args, model, crit, batch, extra = _build(name, dev)
    # each run writes its own stage-2 pseudo-label files
    inputs = _rank_inputs(name, rank, dev, batch, extra, os.path.join(tmp, "ddp"))
    shared = _rank_inputs(name, 0, dev, batch, extra, os.path.join(tmp, "shared"))
    _perturb(model, rank)
    _fix_selection(model, rank)
    model = _convert(model)
    # (a) weight planes packed from this rank's own parameters, then DDP's broadcast of rank 0's
    model.eval()
    with torch.no_grad():
        model(shared, encoder_only=True)
    ddp = DDP(model, device_ids=[0], find_unused_parameters=False)
    with torch.no_grad():
        xyz, feats = ddp(shared, encoder_only=True)
    res["shared_out"] = (xyz.cpu(), feats.cpu())
    model.train()
    if getattr(model, "clip_model", None) is not None:
        model.clip_model.eval()
    params = [p for p in model.parameters() if p.requires_grad]
    opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=0.1)
    res["spread"] = []
    for step in range(STEPS):
        opt.zero_grad()
        out = ddp(inputs, curr_epoch=0)
        loss, _ = crit(out, inputs)
        loss.backward()
        if step == 0:
            res["grads"] = {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.requires_grad}
            res["missing"] = [n for n, p in model.named_parameters() if p.requires_grad and p.grad is None]
            res["stats"] = {n: b.detach().cpu() for n, b in model.named_buffers() if "running_" in n}
        torch.nn.utils.clip_grad_norm_(ddp.parameters(), float(args.clip_gradient))
        opt.step()
        res["spread"].append(_spread(_flat(model)))
    del ddp, model, opt
    # (b) TrainStep(sync_bn=True) on the unconverted model, same ranks and batches
    from coda_neurips2023_b200.engine import TrainStep

    args, model, crit, batch, extra = _build(name, dev)
    inputs = _rank_inputs(name, rank, dev, batch, extra, os.path.join(tmp, "train_step"))
    _perturb(model, rank)
    _fix_selection(model, rank)
    step = TrainStep(args, model, crit, dev, nbuckets=3, sync_bn=True)
    step.prepare(inputs)
    step.flat.zero_grad()
    step.reducer.start()
    step._draw_selection(SCENES_PER_RANK)
    out = model(inputs, curr_epoch=0)
    loss, _ = crit(out, inputs)
    loss.backward()
    step.reducer.finish()
    res["ts_grads"] = {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.requires_grad}
    res["ts_stats"] = {n: b.detach().cpu() for n, b in model.named_buffers() if "running_" in n}
    ops.set_grad_sink(None)
    ops.set_bn_sync(False)
    ops.invalidate_weight_cache()
    dist.barrier()
    return res


def _rank_worker(rank, world, port, outdir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    torch.cuda.set_device(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600))
    tmp = tempfile.mkdtemp(prefix=f"coda_ddp_r{rank}_")
    for name in DDP_CASES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            res = _ddp_case(name, rank, torch.device("cuda", 0), tmp)
        if rank > 0:                     # the other ranks' gradients are rank 0's after the all-reduce (checked: (d))
            res = {k: res[k] for k in ("shared_out", "spread", "missing")}
        torch.save(res, os.path.join(outdir, f"{name}_rank{rank}.pt"))
    torch.save(_evaluate_ddp(rank, world, torch.device("cuda", 0)), os.path.join(outdir, f"evaluate_rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _sampler_shares(world):
    from torch.utils.data import DistributedSampler

    return [list(DistributedSampler(range(ED.NSCENES), num_replicas=world, rank=r, shuffle=False))
            for r in range(world)]


def _evaluate_ddp(rank, world, dev):
    """3.: engine.evaluate on the converted, DDP-wrapped model, this rank's DistributedSampler share of the scenes"""
    from torch.nn.parallel import DistributedDataParallel as DDP

    from coda_neurips2023_b200 import engine, synthetic

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        args, cfg, model, scenes = ED._model_and_data(dev)
    ddp = DDP(_convert(model).eval(), device_ids=[0], find_unused_parameters=False)
    mine = _sampler_shares(world)[rank]
    loader = (synthetic.to_device({k: v[mine[i:i + ED.BATCH]] for k, v in scenes.items()}, dev)
              for i in range(0, len(mine), ED.BATCH))
    return ED._flat(engine.evaluate(args, 0, ddp, None, cfg, loader, if_real_test=True).compute_metrics())


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture(scope="module")
def ddp_ranks(tmp_path_factory):
    import torch.multiprocessing as mp

    outdir = str(tmp_path_factory.mktemp("sync_bn_modules"))
    mp.spawn(_rank_worker, args=(WORLD, _free_port(), outdir), nprocs=WORLD, join=True)
    return outdir


def _load(outdir, name, rank):
    return torch.load(os.path.join(outdir, f"{name}_rank{rank}.pt"))


@pytest.mark.parametrize("name", DDP_CASES)
def test_ddp_on_converted_model_after_the_broadcast(ddp_ranks, name):
    """(a): every rank's forward right after DDP's construction gives rank 0's bits"""
    first = _load(ddp_ranks, name, 0)["shared_out"]
    for r in range(1, WORLD):
        got = _load(ddp_ranks, name, r)["shared_out"]
        for a, b in zip(first, got):
            assert torch.equal(a, b), f"rank {r}'s forward after DDP's broadcast differs from rank 0's"


def _reorder_noise(name):
    """per parameter: the single-process gradient (scene order CONCAT_PERMS[0]) and the largest relative-L2 change of
    it when the scenes are visited in the other orders"""
    ref = _single_process(name, CONCAT_PERMS[0])[0]
    alts = [_single_process(name, p)[0] for p in CONCAT_PERMS[1:]]
    return ref, {n: max(float((a[n] - e).norm()) / max(float(e.norm()), 1e-12) for a in alts) for n, e in ref.items()}


@pytest.mark.parametrize("name", DDP_CASES)
def test_ddp_reference_loop_equals_train_step_sync_bn(ddp_ranks, name):
    """(b) and (d)"""
    res = _load(ddp_ranks, name, 0)
    _, noise = _reorder_noise(name)
    rounding = sorted(n for n, z in noise.items() if z > ROUNDING_NOISE)
    for r in range(WORLD):
        rr = _load(ddp_ranks, name, r)
        assert rr["missing"] == [], f"rank {r}: trainable parameters without a gradient: {rr['missing']}"
        assert rr["spread"] == [0.0] * STEPS, f"rank {r}: parameters differ across ranks after a step: {rr['spread']}"
    assert res["grads"].keys() == res["ts_grads"].keys()
    scale = max(float(e.abs().max()) for e in res["ts_grads"].values())
    worst, worst_name, own, own_name = 0.0, None, 0.0, None
    for n, e in res["ts_grads"].items():
        d = float((res["grads"][n] - e).abs().max())
        if d / scale >= worst:
            worst, worst_name = d / scale, n
        if n not in rounding and d / max(float(e.abs().max()), 1e-30) >= own:
            own, own_name = d / max(float(e.abs().max()), 1e-30), n
    stat = max(float((res["stats"][n].double() - e.double()).abs().max()) for n, e in res["ts_stats"].items())
    print(f"PARITY sync_bn_modules ddp {name}: gradient deviation from TrainStep(sync_bn=True) {worst:.2e} of the "
          f"largest gradient (bar {GRAD_BAR:.0e}, at {worst_name}); {own:.2e} of its own tensor's largest "
          f"(bar {OWN_BAR:.0e}, at {own_name}; pure rounding, global bar only: {', '.join(rounding)}), running statistics {stat:.2e} "
          f"(bar {STATS_BAR:.0e})")
    assert worst <= GRAD_BAR
    assert own <= OWN_BAR
    assert stat <= STATS_BAR


def _single_process(name, perm):
    """rank-summed reference: ONE process, the unconverted model (rank 0's parameters), all WORLD ranks' scenes in
    the order `perm`, BatchNorm in training mode over all the rows -> first-step gradients and running statistics"""
    from coda_neurips2023_b200 import synthetic

    key = (name, tuple(perm))
    if key in _SINGLE:
        return _SINGLE[key]
    perm = np.asarray(perm)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        args, model, crit, batch, extra = _build(name, "cuda")
    # the objectness loss averages over the scenes that hold a box (criterion.py:219-246): with a box in every scene
    # each rank divides by the same count, and the mean over ranks is the concatenated batch's
    assert (batch["gt_box_present"].sum(1) > 0).all()
    sel = np.random.RandomState(5).choice(128, size=(WORLD * SCENES_PER_RANK, 32))[perm]
    model.draw_box_selection = lambda bsz: sel.astype(np.int64)
    inputs = synthetic.to_device({k: v[perm] for k, v in batch.items()}, "cuda")
    if extra.get("pseudo"):
        tmp = tempfile.mkdtemp(prefix="coda_single_")
        inputs["pseudo_box_path"] = [os.path.join(tmp, f"s{i}.npy") for i in range(len(perm))]
    out = model(inputs, curr_epoch=0)
    loss, _ = crit(out, inputs)
    loss.backward()
    grads = {n: p.grad.detach().cpu().double() for n, p in model.named_parameters() if p.requires_grad}
    stats = {n: b.detach().cpu().double() for n, b in model.named_buffers() if "running_" in n}
    _SINGLE[key] = grads, stats
    return grads, stats


_SINGLE: dict = {}      # (case, scene order) -> single-process results, shared by (b) and (c)


@pytest.mark.parametrize("name", CONCAT_CASES)
def test_ddp_reference_loop_equals_one_process_on_the_concatenated_batch(ddp_ranks, name):
    """(c): the DDP path's rank-summed first-step gradients and its running statistics against one process with
    plain BatchNorm on the concatenated batch, each parameter held to a few times its own reorder noise"""
    res = _load(ddp_ranks, name, 0)
    ref, ref_stats = _single_process(name, CONCAT_PERMS[0])
    alts = [_single_process(name, p)[0] for p in CONCAT_PERMS[1:]]
    assert ref.keys() == res["grads"].keys()
    worst, devs = 0.0, []
    for n, e in ref.items():
        norm = max(float(e.norm()), 1e-12)
        dev = float((res["grads"][n].double() - e).norm()) / norm      # relative L2: robust against a single ReLU-mask
        noise = max(float((a[n] - e).norm()) / norm for a in alts)    # flip in a sparse channel
        bar = max(CONCAT_NOISE_FACTOR * noise, CONCAT_FLOOR)
        devs.append((dev / bar, dev, noise, n))
        worst = max(worst, dev / bar)
    devs.sort(reverse=True)
    stat = max(float((res["stats"][n].double() - e).abs().max()) / max(float(e.abs().max()), 1e-6)
               for n, e in ref_stats.items())
    print(f"PARITY sync_bn_modules ddp vs concatenated batch {name}: worst gradient deviation / "
          f"({CONCAT_NOISE_FACTOR:g} x reorder noise, floor {CONCAT_FLOOR:g}) = {worst:.2f} (bar 1), largest: "
          + ", ".join(f"{n} dev {d:.1e} noise {z:.1e}" for _, d, z, n in devs[:3])
          + f"; running statistics {stat:.2e} (bar {CONCAT_STATS_BAR:.0e})")
    assert worst < 1.0
    assert stat < CONCAT_STATS_BAR


def test_engine_evaluate_on_converted_ddp_model_equals_one_process(ddp_ranks):
    """3.: the ranks' metrics are the same, bit for bit, and equal those of engine.evaluate in one process with the
    unconverted model over the stream the reference's all-gather builds (per step rank 0's batch, then rank 1's, ...)"""
    from coda_neurips2023_b200 import engine, synthetic

    got = [torch.load(os.path.join(ddp_ranks, f"evaluate_rank{r}.pt")) for r in range(WORLD)]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        args, cfg, model, scenes = ED._model_and_data("cuda")
    shares = _sampler_shares(WORLD)
    stream = []
    for s in range(0, len(shares[0]), ED.BATCH):
        idx = [i for r in range(WORLD) for i in shares[r][s:s + ED.BATCH]]
        stream.append(synthetic.to_device({k: v[idx] for k, v in scenes.items()}, "cuda"))
    want = ED._flat(engine.evaluate(args, 0, model, None, cfg, stream, if_real_test=True).compute_metrics())
    for r in range(1, WORLD):
        ED._close_flat(got[r], got[0], 0.0)
    dev = max((abs(a - b) for thr in want for (_, a), (_, b) in zip(got[0][thr], want[thr])
               if not (np.isnan(a) and np.isnan(b))), default=0.0)
    print(f"PARITY sync_bn_modules evaluate on {WORLD} gloo ranks (converted, DDP) vs one process (unconverted): "
          f"max metric deviation {dev:.2e} (bar 1e-5), ranks bit-identical")
    ED._close_flat(got[0], want, 1e-5)
