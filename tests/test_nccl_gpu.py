"""Data-parallel step over NCCL on 2 GPUs of one box (skipped on a single-GPU box): what engine.TrainStep promises.

  * ranks are seeded DIFFERENTLY (reference main.py:982-985): the rank-0 broadcast in TrainStep.prepare must make
    the replicas identical;
  * the bucketed, overlapped all-reduce (hooks + direct gradient writes, inside the CUDA graph) must give every rank
    the MEAN of the two ranks' gradients: with BatchNorm in eval mode (per-GPU statistics are the one thing that is
    not data-parallel-equivalent) and scenes that are the two halves of one batch, the flat gradient of each rank
    equals the gradient of the same model on the CONCATENATED batch on one GPU (losses are normalised by the
    all-reduced box count, criterion.py:1180-1186);
  * after a few optimiser steps both ranks hold bit-identical weights."""
import os
import socket
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _build(seed, args):
    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.models import build_model

    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    return model, build_criterion(args, cfg)


def _bn_eval(model):
    for m in model.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.eval()


def _args():
    from coda_neurips2023_b200 import synthetic

    return synthetic.make_args(nqueries=128, preenc_npoints=256, dec_dim=128, dec_nlayers=2, dec_ffn_dim=64,
                               enc_dropout=0.0, dec_dropout=0.0, mlp_dropout=0.0, ngpus=2,
                               # this loss is normalised by the LOCAL number of valid crops (criterion.py:924-943), so
                               # the mean over ranks is not the loss of the concatenated batch: keep it out of the check
                               loss_predicted_region_embed_l1_weight=0.0)


def _worker(rank, world, port, ret, sync_bn=False):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.engine import TrainStep

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    args = _args()
    model, crit = _build(100 + rank, args)            # different initialisation per rank
    model = model.to(dev).train()
    model.clip_model.eval()
    if not sync_bn:
        _bn_eval(model)
    crit = crit.to(dev)
    full = synthetic.make_batch(4, 3000, seed=7)
    mine = {k: v[rank * 2: rank * 2 + 2] for k, v in full.items()}
    batch = synthetic.to_device(mine, dev)
    sel = np.random.RandomState(5).choice(128, size=(4, 32))      # the same crop boxes as the single-GPU run
    model.draw_box_selection = lambda bsz: sel[rank * 2: rank * 2 + 2].astype(np.int64)
    step = TrainStep(args, model, crit, dev, nbuckets=3, sync_bn=sync_bn)
    step.prepare(batch)
    w0 = step.flat.flat_param.detach().clone()
    # one eager backward through the step body WITHOUT the optimiser: capture the reduced gradient
    step.flat.zero_grad()
    step.reducer.start()
    out = model(batch, curr_epoch=0)
    loss, _ = crit(out, batch)
    loss.backward()
    launched_early = sum(step.reducer.launched)
    step.reducer.finish()
    grads = {n: p.grad.detach().clone().cpu() for n, p in model.named_parameters() if p.requires_grad}
    if rank == 0:
        ret["loss"] = float(loss)
        ret["bn_mean"] = {n: b.detach().clone().cpu() for n, b in model.named_buffers() if n.endswith("running_mean")}
    # drop the eager graph: its AccumulateGrad nodes were created on the default stream and would be reused (with
    # that stream) by the capture below
    del out, loss
    # then a few real steps (eager here; the CUDA-graph-captured form of the same body, NCCL ranges included, is
    # what bench.py --gpus 2 runs and checks with `param_spread_across_ranks`)
    for _ in range(3):
        step(batch, 0.0)
    torch.cuda.synchronize()
    w = step.flat.flat_param.detach().clone()
    hi, lo = w.clone(), w.clone()
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    w0hi = w0.clone()
    dist.all_reduce(w0hi, op=dist.ReduceOp.MAX)
    if rank == 0:
        ret["spread_after_steps"] = float((hi - lo).abs().max())
        ret["spread_after_broadcast"] = float((w0hi - w0).abs().max())
        ret["moved"] = float((w - w0).abs().max())
        ret["grads"] = grads
        ret["launched_early"] = launched_early
        ret["nranges"] = len(step.reducer.ranges)
    dist.barrier()
    os._exit(0)       # a live CUDA graph references the communicator: do not tear NCCL down


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_step_equals_concatenated_batch(built_lib):
    import torch.multiprocessing as mp

    from coda_neurips2023_b200 import synthetic

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    assert ret["spread_after_broadcast"] == 0.0, "rank 0's parameters were not broadcast"
    assert ret["spread_after_steps"] == 0.0, "ranks diverged"
    assert ret["moved"] > 0
    assert ret["nranges"] == 3 and ret["launched_early"] >= 1, "no range all-reduce started during the backward"
    # single GPU, rank 0's initialisation, the whole batch
    args = _args()
    args.ngpus = 1
    model, crit = _build(100, args)
    model = model.cuda().train()
    model.clip_model.eval()
    _bn_eval(model)
    crit = crit.cuda()
    sel = np.random.RandomState(5).choice(128, size=(4, 32))
    model.draw_box_selection = lambda bsz: sel.astype(np.int64)
    batch = synthetic.to_device(synthetic.make_batch(4, 3000, seed=7), "cuda")
    out = model(batch, curr_epoch=0)
    loss, _ = crit(out, batch)
    loss.backward()
    worst = 0.0
    for n, p in model.named_parameters():
        if p.requires_grad and p.grad is not None:
            g, e = ret["grads"][n].double(), p.grad.detach().cpu().double()
            scale = max(float(e.abs().max()), 1e-5)
            worst = max(worst, float((g - e).abs().max()) / scale)
    print(f"PARITY nccl_2rank: max relative deviation of the all-reduced gradient from the 1-GPU gradient {worst:.2e}")
    assert worst < 2e-2     # 2 bf16 planes in the backward, different reduction orders


def _single_gpu_train_bn_grads(perm):
    """gradient and BatchNorm running means of ONE GPU on the 4-scene batch (BatchNorm in training mode), scenes
    visited in the order `perm`: mathematically the same batch, a different order of every reduction"""
    from coda_neurips2023_b200 import synthetic

    args = _args()
    args.ngpus = 1
    model, crit = _build(100, args)
    model = model.cuda().train()
    model.clip_model.eval()
    crit = crit.cuda()
    sel = np.random.RandomState(5).choice(128, size=(4, 32))[perm]
    model.draw_box_selection = lambda bsz: sel.astype(np.int64)
    full = synthetic.make_batch(4, 3000, seed=7)
    batch = synthetic.to_device({k: v[perm] for k, v in full.items()}, "cuda")
    out = model(batch, curr_epoch=0)
    loss, _ = crit(out, batch)
    loss.backward()
    grads = {n: p.grad.detach().cpu().double() for n, p in model.named_parameters() if p.requires_grad and p.grad is not None}
    means = {n: b.detach().cpu().double() for n, b in model.named_buffers() if n.endswith("running_mean")}
    return grads, means


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_sync_batchnorm_equals_concatenated_batch(built_lib):
    """TrainStep(sync_bn=True): BatchNorm in TRAINING mode with statistics all-reduced over the ranks (the
    reference's convert_sync_batchnorm, main.py:993).  Two ranks x 2 scenes must then give the gradient -- and the
    running statistics -- of one GPU on the 4-scene batch: the SyncBN exchange (fp64 column sums forward, averaged
    (sum dz, sum dz xhat) backward, 18 layers) is what makes data parallelism batch-equivalent.

    Training-mode BatchNorm subtracts batch means in its backward, which amplifies the rounding of the two-plane
    gradient GEMMs by the cancellation factor (a LayerNorm bias in front of a Linear + BatchNorm has a gradient that is
    zero in exact arithmetic: what is measured there is pure rounding).  The yardstick is therefore measured, not
    assumed: the same single-GPU batch with its scenes in another order -- identical mathematics, another order of
    every reduction -- and each parameter is held to a few times ITS OWN noise."""
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), ret, True), nprocs=2, join=True)
    assert ret["spread_after_steps"] == 0.0, "ranks diverged"
    ref, ref_means = _single_gpu_train_bn_grads(np.array([0, 1, 2, 3]))
    alts = [_single_gpu_train_bn_grads(np.array(p))[0] for p in ([2, 3, 0, 1], [1, 0, 3, 2], [3, 2, 1, 0])]
    devs, worst_excess = [], 0.0
    for n, e in ref.items():
        norm = max(float(e.norm()), 1e-7)
        dev = float((ret["grads"][n].double() - e).norm()) / norm             # relative L2: robust against a single
        noise = max(float((a[n] - e).norm()) / norm for a in alts)             # ReLU-mask flip in a sparse channel
        devs.append((dev, noise, n))
        worst_excess = max(worst_excess, dev / max(6.0 * noise, 3e-3))
    devs.sort(reverse=True)
    stat = max(float((ret["bn_mean"][n].double() - e).abs().max()) / max(float(e.abs().max()), 1e-6)
               for n, e in ref_means.items())
    print("largest relative-L2 gradient deviations (2 ranks vs 1 GPU | same GPU, scenes reordered, max of 3):",
          [(f"{d:.1e}", f"{z:.1e}", n) for d, z, n in devs[:6]])
    for d, z, n in devs:
        if d > max(6.0 * z, 3e-3):
            print(f"  OUTLIER {n}: dev {d:.2e} noise {z:.2e}")
    print(f"PARITY nccl_2rank_syncbn: worst deviation / (6 x reorder noise, floor 3e-3) = {worst_excess:.2f}, "
          f"running-mean deviation {stat:.2e}")
    assert stat < 1e-4
    assert worst_excess < 1.0
