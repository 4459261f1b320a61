"""TrainStep's captured step on a model converted by convert_sync_batchnorm, over NCCL on 2 GPUs of one box (skipped on
a single-GPU box).

The converted model's nn.SyncBatchNorm modules synchronise over their process group whatever `sync_bn` says
(ops.bn_sync_group).  So TrainStep(sync_bn=False).capture on the converted model must run the step of
TrainStep(sync_bn=True).capture on the unconverted model: the same collectives on the same sums, inside the CUDA
graph.  Both start from the same rank-0 parameters and replay two steps on the same per-rank batches."""
import os
import socket
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

REPLAYS = 2
BAR = 1e-6         # max |difference| / max |parameter| of the flat parameters after REPLAYS replayed steps


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _args():
    from coda_neurips2023_b200 import synthetic

    return synthetic.make_args(nqueries=128, preenc_npoints=256, dec_dim=128, dec_nlayers=2, dec_ffn_dim=64,
                               enc_dropout=0.0, dec_dropout=0.0, mlp_dropout=0.0, ngpus=2)


def _flat_after_replays(rank, dev, convert, batch):
    from coda_neurips2023_b200 import ops, synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.engine import TrainStep
    from coda_neurips2023_b200.models import build_model

    args = _args()
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(100 + rank)                   # different initialisation per rank: the step broadcasts rank 0's
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model = model.to(dev).train()
    model.clip_model.eval()
    if convert:
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    crit = build_criterion(args, cfg).to(dev)
    sel = np.random.RandomState(5).choice(128, size=(4, 32))
    model.draw_box_selection = lambda bsz: sel[rank * 2: rank * 2 + 2].astype(np.int64)
    step = TrainStep(args, model, crit, dev, nbuckets=3, sync_bn=not convert)
    step.capture(batch)
    for _ in range(REPLAYS):
        step(batch, 0.0)
    torch.cuda.synchronize()
    names = list(step.flat.names)
    flat = {n: p.detach().cpu().clone() for n, p in zip(names, step.flat.params)}
    ops.set_grad_sink(None)
    ops.set_bn_sync(False)
    return flat, step


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    from coda_neurips2023_b200 import synthetic

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    full = synthetic.make_batch(4, 3000, seed=7)
    batch = synthetic.to_device({k: v[rank * 2: rank * 2 + 2] for k, v in full.items()}, dev)
    plain, keep_a = _flat_after_replays(rank, dev, False, batch)
    converted, keep_b = _flat_after_replays(rank, dev, True, batch)
    if rank == 0:
        ret["plain"], ret["converted"] = plain, converted
    dist.barrier()
    os._exit(0)       # live CUDA graphs reference the communicator: do not tear NCCL down


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_captured_step_on_converted_model_equals_sync_bn_on_unconverted(built_lib):
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    plain, converted = ret["plain"], ret["converted"]
    assert plain.keys() == converted.keys()
    worst = max(float((converted[n] - e).abs().max()) / max(float(e.abs().max()), 1e-12) for n, e in plain.items())
    print(f"PARITY sync_bn_modules nccl capture: converted vs sync_bn=True after {REPLAYS} replays {worst:.2e} "
          f"(bar {BAR:.0e})")
    assert worst <= BAR
