"""Data-parallel evaluation (coda_neurips2023_b200/utils/ap_calculator.py, include/coda_eval.h):

  * `coda_eval_ap` against fp64 numpy (utils/eval_det.py:147-162, voc_ap) per class and IoU threshold;
  * `coda_eval_records` against a numpy enumeration of the stored step tensors;
  * W simulated ranks, each a rank-local calculator over its contiguous slice of every step, merged by
    `merge_rank_states`: the metrics must equal, bit for bit, those of one calculator stepped on the whole batches;
  * the reference golden (tests/golden/eval_ap.npz) reproduced from two simulated ranks;
  * the collective of a rank-local `compute_metrics()` itself, on three gloo ranks sharing one GPU, with an empty rank
    and a one-record rank;
  * two NCCL ranks through `engine.evaluate` (needs 2 GPUs)."""
import datetime
import os
import socket
import warnings
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from coda_neurips2023_b200.utils import ap_calculator as apc
from coda_neurips2023_b200.utils.box_util import flip_axis_to_camera_tensor, get_3d_box_batch_tensor

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "eval_ap.npz"


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


# --------------------------------------------------------------------------- coda_eval_ap
def _numpy_class(tp_bits, npos):
    """utils/eval_det.py:147-162 + voc_ap on one class's sorted true-positive flags"""
    tp = np.cumsum(tp_bits.astype(np.float64))
    fp = np.cumsum(1.0 - tp_bits.astype(np.float64))
    rec = np.zeros_like(tp) if npos == 0 else tp / float(npos)
    prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
    return tp, fp, rec, prec, apc.voc_ap(rec, prec)


def test_eval_ap_equals_numpy_voc_ap():
    rng = np.random.default_rng(0)
    nthr = 2
    # per class: (records, true-positive probability, npos beyond the true positives)
    spec = [(1, 1.0, 0), (1, 0.0, 2), (200_000, 0.3, 5000), (64, 1.0, 0), (64, 1.0, 10), (48, 0.0, 7), (33, 0.5, None),
            (0, 0.0, 9), (0, 0.0, 0), (5000, 0.05, 1), (3000, 0.9, 0)]
    cls, tp, npos = [], [], []
    for c, (n, p, extra) in enumerate(spec):
        bits = (rng.random((nthr, n)) < p).astype(np.uint32)
        if n > 10:
            bits[1] &= bits[0]                      # the stricter threshold keeps a subset of the matches
        cls.append(np.full(n, c, np.int32))
        tp.append(bits[0] | (bits[1] << 1))
        # npos = 0 with detections: every detection of that class is a false positive
        npos.append(0 if extra is None else int(bits.sum(1).max()) + extra)
        if extra is None:
            tp[-1][:] = 0
    ncls = len(spec)
    cls = np.concatenate(cls)
    tpm = np.concatenate(tp)
    rec = apc.EvalRecords(torch.from_numpy(cls).cuda(), torch.zeros(len(cls), device="cuda"),
                          torch.zeros(len(cls), dtype=torch.int64, device="cuda"),
                          torch.from_numpy(tpm.view(np.int32)).cuda())
    ap, last_prec, last_rec, counts, curves = apc.eval_ap(rec, ncls, nthr, torch.tensor(npos, device="cuda"), curves=True)
    ap, last_prec, last_rec, curves = (x.cpu().numpy() for x in (ap, last_prec, last_rec, curves))
    assert counts.cpu().tolist() == [s[0] for s in spec]
    lo = 0
    worst = 0.0
    for c, (n, _, _) in enumerate(spec):
        for t in range(nthr):
            bits = (tpm[lo:lo + n] >> t) & 1
            etp, efp, erec, eprec, eap = _numpy_class(bits, npos[c])
            got = curves[t, :, lo:lo + n]
            assert np.array_equal(got[0], etp) and np.array_equal(got[1], efp), (c, t)
            assert np.array_equal(got[2], erec) and np.array_equal(got[3], eprec), (c, t)
            assert abs(ap[t, c] - eap) <= 1e-12, (c, t, ap[t, c], eap)
            worst = max(worst, abs(ap[t, c] - eap))
            assert last_prec[t, c] == (eprec[-1] if n else 0.0) and last_rec[t, c] == (erec[-1] if n else 0.0)
        lo += n
    print(f"PARITY eval_ap: max |AP - numpy voc_ap| = {worst:.1e} over {ncls} classes x {nthr} thresholds")


# --------------------------------------------------------------------------- coda_eval_records
def test_eval_records_equal_numpy_enumeration():
    rng = np.random.default_rng(1)
    k, ncls, nthr = 37, 9, 2
    steps, expect, base = [], set(), 0
    for b in (3, 5):
        s = rng.random((b, k, ncls)).astype(np.float32)
        s[rng.random(s.shape) < 0.2] = -np.inf
        s[rng.random(s.shape) < 0.05] = np.nan
        s[rng.random(s.shape) < 0.02] = np.inf
        s[rng.random(s.shape) < 0.02] = -0.0
        s[rng.random(s.shape) < 0.05] = 0.5                  # ties
        m = rng.random((b, k)) < 0.7
        tp = rng.random((nthr, b, ncls, k)) < 0.3
        steps.append((torch.from_numpy(s).cuda(), torch.from_numpy(m).cuda(), torch.from_numpy(tp).cuda(), base))
        for bb, j, c in zip(*np.nonzero(m[:, :, None] & np.isfinite(s))):
            mask = sum(int(tp[t, bb, c, j]) << t for t in range(nthr))
            expect.add((int(c), float(s[bb, j, c]) + 0.0, (base + int(bb)) * k + int(j), mask))
        base += b + 4                                         # scene numbers need not be contiguous across steps
    rec = apc.eval_records(*(list(x) for x in zip(*steps)))
    got = list(zip(rec.cls.cpu().tolist(), rec.score.cpu().tolist(), rec.pos.cpu().tolist(), rec.tp.cpu().tolist()))
    assert len(got) == len(expect) and set(got) == expect
    assert not any(np.signbit(rec.score.cpu().numpy())), "a zero score must be written as +0"


# --------------------------------------------------------------------------- simulated ranks
def _scenes(seed, n, k=24, ncls=6, g=6, tie_levels=4):
    """n synthetic scenes: ground-truth boxes, predictions around them and elsewhere; class probabilities and
    objectness on a coarse grid so that many scores tie exactly, within and across scenes."""
    rng = np.random.default_rng(seed)
    ctr = rng.uniform(-2, 2, (n, g, 3))
    size = rng.uniform(0.4, 1.5, (n, g, 3))
    ang = rng.uniform(-np.pi, np.pi, (n, g))
    present = rng.random((n, g)) < 0.8
    gcls = rng.integers(0, ncls, (n, g))
    src = rng.integers(0, g, (n, k))
    near = rng.random((n, k)) < 0.6
    pctr = np.where(near[..., None], np.take_along_axis(ctr, src[..., None], 1) + rng.normal(0, 0.15, (n, k, 3)),
                    rng.uniform(-2, 2, (n, k, 3)))
    psize = np.where(near[..., None], np.take_along_axis(size, src[..., None], 1) * rng.uniform(0.8, 1.2, (n, k, 3)),
                     rng.uniform(0.4, 1.5, (n, k, 3)))
    pang = np.where(near, np.take_along_axis(ang, src, 1), rng.uniform(-np.pi, np.pi, (n, k)))
    probs = rng.integers(1, tie_levels + 1, (n, k, ncls)) / tie_levels
    probs[near] += 2.0 * (np.arange(ncls) == np.take_along_axis(gcls, src, 1)[near][:, None])
    obj = rng.integers(0, tie_levels + 1, (n, k)) / tie_levels

    def corners(c, s, a):
        t = lambda x: torch.from_numpy(np.asarray(x, np.float32))  # noqa: E731
        return get_3d_box_batch_tensor(t(s), t(a), flip_axis_to_camera_tensor(t(c)))

    return dict(box_corners=corners(pctr, psize, pang), sem_cls_prob=torch.from_numpy(probs.astype(np.float32)),
                objectness_prob=torch.from_numpy(obj.astype(np.float32)),
                point_clouds=torch.from_numpy(rng.uniform(-2, 2, (n, 64, 3)).astype(np.float32)),
                gt_box_corners=corners(ctr, size, ang), gt_box_sem_cls_label=torch.from_numpy(gcls),
                gt_box_present=torch.from_numpy(present.astype(np.float32)))


def _step(calc, batch):
    batch = {key: v.cuda() for key, v in batch.items()}
    calc.step_meter({"outputs": {key: batch[key] for key in ("box_corners", "sem_cls_prob", "objectness_prob")}},
                    {key: batch[key] for key in ("point_clouds", "gt_box_corners", "gt_box_sem_cls_label",
                                                 "gt_box_present")})


def _slice(batch, lo, hi):
    return {key: v[lo:hi] for key, v in batch.items()}


def _calc(ds, cfg, args, **kw):
    return apc.APCalculator(ds, ap_iou_thresh=[0.25, 0.5], exact_eval=False, args=args, ap_config_dict=cfg, **kw)


def _same(a, b):
    """same keys in the same order, same values bit for bit"""
    assert list(a) == list(b)
    for thr in a:
        assert list(a[thr].keys()) == list(b[thr].keys()), thr
        for key in a[thr]:
            x, y = np.float64(a[thr][key]), np.float64(b[thr][key])
            assert x.tobytes() == y.tobytes() or (np.isnan(x) and np.isnan(y)), (thr, key, x, y)


def _case(name, w, bl=2, nsteps=3):
    """-> per-step whole batches (w * bl scenes, rank r owning scenes r * bl ... r * bl + bl - 1), config, args, ds"""
    ncls = 24 if name == "scannet" else 6
    per_class = name not in ("first_on_rank1", "agnostic", "one_record")
    ds = SimpleNamespace(num_semcls=ncls)
    args = SimpleNamespace(dataset_name="sunrgbd")
    if name == "scannet":
        ds.seen_idx_list, ds.novel_idx_list = list(range(0, 20, 2)), list(range(1, 20, 2)) + [20, 21, 22, 23]
        args = SimpleNamespace(dataset_name="scannet")
    cfg = apc.get_ap_config_dict(dataset_config=ds, remove_empty_box=False, per_class_proposal=per_class,
                                 cls_nms=name != "agnostic")
    steps = []
    for s in range(nsteps):
        batch = _scenes(100 * s + w, w * bl, ncls=ncls, g=12 if name == "scannet" else 6)
        if name == "ties" and w > 1:
            # rank 1's scenes repeat rank 0's predictions exactly, against other ground truth: equal scores across
            # ranks with different true-positive flags, which only the (scene, box) order can rank
            for key in ("box_corners", "sem_cls_prob", "objectness_prob"):
                batch[key][bl:2 * bl] = batch[key][:bl]
        if name == "first_on_rank1":
            # class 4 is predicted on rank 1 in the first step and on rank 0 only from the second on
            batch["sem_cls_prob"][:, :, 4] = 0.0
            owner = slice(bl, 2 * bl) if s == 0 else slice(0, bl)
            batch["sem_cls_prob"][owner, :3, 4] = 9.0
            batch["objectness_prob"][owner, :3] = 1.0
        if name in ("empty_rank", "one_record"):
            batch["objectness_prob"][(w - 1) * bl:] = 0.0       # below conf_thresh: the last rank detects nothing
            batch["gt_box_present"][(w - 1) * bl:] = 0.0
        if name == "one_record":
            # rank 1 (the last rank when w = 2) detects one box in all: one record over the whole evaluation
            batch["objectness_prob"][bl:2 * bl] = 0.0
            if s == 0:
                batch["objectness_prob"][bl, 0] = 1.0
        steps.append(batch)
    return steps, cfg, args, ds


CASES = ["ties", "first_on_rank1", "empty_rank", "one_record", "agnostic", "scannet"]


@pytest.mark.parametrize("w", [2, 3])
@pytest.mark.parametrize("name", CASES)
def test_simulated_ranks_equal_one_calculator(name, w):
    bl = 2
    steps, cfg, args, ds = _case(name, w, bl)
    whole = _calc(ds, cfg, args)
    ranks = [_calc(ds, cfg, args, rank=r, world_size=w) for r in range(w)]
    for batch in steps:
        _step(whole, batch)
        for r, calc in enumerate(ranks):
            _step(calc, _slice(batch, r * bl, (r + 1) * bl))
    assert [c.scan_cnt for c in ranks] == [whole.scan_cnt] * w
    states = [c.rank_state() for c in ranks]
    if name in ("empty_rank", "one_record"):
        assert len(states[-1].records) == (1 if name == "one_record" and w == 2 else 0)
    if name == "one_record":
        assert len(states[1].records) == 1
    merged = apc.merge_rank_states(states)
    got, want = ranks[0].metrics_from_state(merged), whole.compute_metrics()
    _same(got, want)
    classes = [key for key in want[0.25] if key.endswith("Average Precision")]
    if name == "scannet":
        assert len(classes) >= 21 and "mAP_novel" in want[0.25]
    if name == "first_on_rank1":
        k = steps[0]["objectness_prob"].shape[1]
        assert bl <= int(merged.first_pred[4]) // k < 2 * bl          # first seen on rank 1, in the first step
        assert int(states[0].first_pred[4]) // k >= w * bl            # rank 0 sees it in the second step
    # the single-rank path through compute_metrics() is the same computation
    _same(ranks[0].metrics_from_state(whole.rank_state()), want)


@pytest.mark.parametrize("name", ["default", "agnostic", "bev"])
def test_golden_split_over_two_ranks(name):
    """tests/golden/eval_ap.npz (the reference's APCalculator on 2 steps of 2 scenes): every step split over two
    simulated ranks of one scene each reproduces the reference's metrics within test_eval_gpu.py's bar."""
    configs = {"default": dict(), "agnostic": dict(cls_nms=False, per_class_proposal=False, conf_thresh=0.3),
               "bev": dict(use_3d_nms=False, per_class_proposal=False, use_cls_confidence_only=True,
                           remove_empty_box=False)}
    g = np.load(GOLDEN)
    t = {key[3:]: torch.from_numpy(g[key]) for key in g.files if key.startswith("in.")}
    ds = SimpleNamespace(num_semcls=t["sem_cls_prob"].shape[-1])
    cfg = apc.get_ap_config_dict(dataset_config=ds, **configs[name])
    ranks = [apc.APCalculator(ds, ap_iou_thresh=[0.25, 0.5], exact_eval=True, args=SimpleNamespace(dataset_name="sunrgbd"),
                              ap_config_dict=cfg, rank=r, world_size=2) for r in range(2)]
    for lo in (0, 2):
        for r, calc in enumerate(ranks):
            _step(calc, _slice(t, lo + r, lo + r + 1))
    ret = ranks[1].metrics_from_state(apc.merge_rank_states([c.rank_state() for c in ranks]))
    for thr in (0.25, 0.5):
        keys, vals = list(g[f"{name}.{thr}.keys"]), g[f"{name}.{thr}.values"]
        assert set(keys) == set(ret[thr].keys())
        for key, v in zip(keys, vals):
            got = float(ret[thr][key])
            assert (np.isnan(v) and np.isnan(got)) or abs(got - float(v)) < 1e-5, (thr, key, got, float(v))


def test_unequal_batch_sizes_across_ranks_raise():
    steps, cfg, args, ds = _case("ties", 2, 2, nsteps=2)
    ranks = [_calc(ds, cfg, args, rank=r, world_size=2) for r in range(2)]
    _step(ranks[0], _slice(steps[0], 0, 2))
    _step(ranks[1], _slice(steps[0], 2, 4))
    _step(ranks[0], _slice(steps[1], 0, 2))
    _step(ranks[1], _slice(steps[1], 2, 3))                 # one scene short on rank 1
    with pytest.raises(ValueError):
        apc.merge_rank_states([c.rank_state() for c in ranks])


# --------------------------------------------------------------------------- two NCCL ranks
NSCENES, BATCH = 12, 2


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _model_and_data(device):
    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(nqueries=64, preenc_npoints=256, dec_dim=128, dec_nlayers=2, dec_ffn_dim=64)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    scenes = synthetic.make_batch(NSCENES, 3000, seed=11)
    return args, cfg, model.to(device).eval(), scenes


def _flat(ret):
    return {thr: [(key, float(v)) for key, v in d.items()] for thr, d in ret.items()}


def _eval_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    from torch.utils.data import DataLoader, DistributedSampler

    from coda_neurips2023_b200 import engine, synthetic

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    args, cfg, model, scenes = _model_and_data(dev)
    items = [{key: v[i] for key, v in scenes.items()} for i in range(NSCENES)]
    sampler = DistributedSampler(items, num_replicas=world, rank=rank, shuffle=False)
    loader = (synthetic.to_device(b, dev) for b in DataLoader(items, batch_size=BATCH, sampler=sampler,
                                                             collate_fn=_collate))
    calc = engine.evaluate(args, 0, model, None, cfg, loader, if_real_test=True)
    ret = calc.compute_metrics()
    out[rank] = _flat(ret)
    dist.barrier()
    dist.destroy_process_group()


def _collate(items):
    return {key: np.stack([it[key] for it in items]) for key in items[0]}


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_engine_evaluate_equals_gathered_stream():
    """engine.evaluate on 2 NCCL ranks, each fed its DistributedSampler share, returns on both ranks the metrics of
    engine.evaluate in one process over the stream the reference's all-gather builds (per step rank 0's batch, then
    rank 1's)."""
    import torch.multiprocessing as mp

    from coda_neurips2023_b200 import engine, synthetic

    w = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_eval_worker, args=(w, _free_port(), out), nprocs=w, join=True)
    args, cfg, model, scenes = _model_and_data("cuda")
    per_rank = [list(range(r, NSCENES, w)) for r in range(w)]
    stream = []
    for s in range(0, NSCENES // w, BATCH):
        idx = [i for r in range(w) for i in per_rank[r][s:s + BATCH]]
        stream.append(synthetic.to_device({key: v[idx] for key, v in scenes.items()}, "cuda"))
    want = _flat(engine.evaluate(args, 0, model, None, cfg, stream, if_real_test=True).compute_metrics())
    _close_flat(out[1], out[0], 0.0)
    _close_flat(out[0], want, 1e-5)


def _close_flat(got, want, tol):
    """same thresholds and keys in the same order, values within tol (tol = 0: bit for bit); NaN matches NaN"""
    assert list(got) == list(want)
    for thr in want:
        assert [key for key, _ in got[thr]] == [key for key, _ in want[thr]], thr
        for (key, a), (_, b) in zip(got[thr], want[thr]):
            same = np.float64(a).tobytes() == np.float64(b).tobytes() if tol == 0 else abs(a - b) <= tol
            assert same or (np.isnan(a) and np.isnan(b)), (thr, key, a, b)


def _gloo_worker(rank, world, port, name, bl, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    steps, cfg, args, ds = _case(name, world, bl)
    calc = _calc(ds, cfg, args, rank=rank, world_size=world)
    for batch in steps:
        _step(calc, _slice(batch, rank * bl, (rank + 1) * bl))
    out[f"records{rank}"] = len(calc.rank_state().records)
    out[rank] = _flat(calc.compute_metrics())
    dist.destroy_process_group()


@pytest.mark.parametrize("name", ["one_record", "empty_rank"])
def test_collective_compute_metrics_gloo_ranks_on_one_gpu(name):
    """The collective a rank-local compute_metrics() runs (batch sizes, record exchange, SUM / MIN all-reduces), on
    three gloo ranks sharing one GPU, with a rank that holds no record (and one that holds a single record): every
    rank gets, bit for bit, the metrics of one calculator stepped on the whole batches."""
    import torch.multiprocessing as mp

    w, bl = 3, 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_gloo_worker, args=(w, _free_port(), name, bl, out), nprocs=w, join=True)
    counts = [out[f"records{r}"] for r in range(w)]
    assert counts[2] == 0 and (counts[1] == 1 if name == "one_record" else counts[1] > 1), counts
    steps, cfg, args, ds = _case(name, w, bl)
    whole = _calc(ds, cfg, args)
    for batch in steps:
        _step(whole, batch)
    want = _flat(whole.compute_metrics())
    for r in range(w):
        _close_flat(out[r], want, 0.0)
