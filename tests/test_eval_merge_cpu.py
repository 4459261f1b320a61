"""Host side of data-parallel evaluation (coda_neurips2023_b200/utils/ap_calculator.py), without a GPU:

  * `sort_records` against numpy's lexicographic sort: class ascending, score descending (-0 ties with +0), global
    (scene, box) position ascending;
  * `pack_records` / `unpack_records` through the padded exchange buffer, at 0, 1 and several records per rank;
  * the collective behind a rank-local `compute_metrics()` (`APCalculator._all_rank_state`) on three gloo ranks
    holding 5, 0 and 1 records: every rank must end with `merge_rank_states` of the three states, and unequal batch
    sizes must raise ValueError on every rank."""
import datetime
import os
import socket
from types import SimpleNamespace

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from coda_neurips2023_b200.utils import ap_calculator as apc

NCLS = 7
BIG = torch.iinfo(torch.int64).max


def _records(seed, n):
    rng = np.random.default_rng(seed)
    score = rng.choice(np.array([0.5, 0.25, -0.0, 0.0, -1.5, 3.0, 1e-30], np.float32), n)
    return apc.EvalRecords(torch.from_numpy(rng.integers(0, NCLS, n).astype(np.int32)), torch.from_numpy(score),
                           torch.from_numpy(rng.permutation(n * 3)[:n].astype(np.int64) + (1 << 33)),
                           torch.from_numpy(rng.integers(0, 4, n).astype(np.int32)))


def test_sort_records_equals_lexsort():
    rec = _records(0, 20_000)
    got = apc.sort_records(rec)
    s = rec.score.numpy().astype(np.float64) + 0.0
    order = np.lexsort((rec.pos.numpy(), -s, rec.cls.numpy()))
    for name, g, r in zip(rec._fields, got, rec):
        assert np.array_equal(g.numpy().view(np.int32) if name == "score" else g.numpy(),
                              r.numpy()[order].view(np.int32) if name == "score" else r.numpy()[order]), name


def test_pack_unpack_through_padded_buffer():
    for n in (0, 1, 2, 5):
        rec = _records(n, n)
        buf = torch.zeros((6, 5), dtype=torch.int32)
        buf[:n] = apc.pack_records(rec)
        back = apc.unpack_records(buf[:n])
        for name, a, b in zip(rec._fields, back, rec):
            assert a.dtype == b.dtype and torch.equal(a.view(torch.int32) if name == "score" else a,
                                                      b.view(torch.int32) if name == "score" else b), (n, name)


def _state(rank, batch_sizes):
    n = (5, 0, 1)[rank]
    g = torch.Generator().manual_seed(rank)
    first = torch.randint(0, 1000, (NCLS,), generator=g)
    first[rank] = BIG                                           # never seen on this rank
    return apc.RankState(_records(10 + rank, n), torch.randint(0, 4, (NCLS,), generator=g), first,
                         torch.randint(0, 1000, (NCLS,), generator=g), batch_sizes)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    calc = apc.APCalculator(SimpleNamespace(num_semcls=NCLS), rank=rank, world_size=world)
    merged = calc._all_rank_state(_state(rank, [2, 2, 1]))
    ret[rank] = [t.clone() for t in (*merged.records, merged.gt_count, merged.first_pred, merged.first_gt)]
    try:
        calc._all_rank_state(_state(rank, [2, 2 if rank != 1 else 1]))
        ret[f"raised{rank}"] = False
    except ValueError:
        ret[f"raised{rank}"] = True
    dist.destroy_process_group()


def test_collective_merge_with_empty_and_one_record_ranks_gloo():
    world = 3
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    want = apc.merge_rank_states([_state(r, [2, 2, 1]) for r in range(world)])
    want = [*want.records, want.gt_count, want.first_pred, want.first_gt]
    for r in range(world):
        assert len(ret[r][0]) == 6
        for a, b in zip(ret[r], want):
            assert a.dtype == b.dtype and torch.equal(a.view(torch.int32) if a.is_floating_point() else a,
                                                      b.view(torch.int32) if b.is_floating_point() else b), r
        assert ret[f"raised{r}"], f"rank {r} did not refuse unequal batch sizes"
