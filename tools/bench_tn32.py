"""Time the weight-gradient GEMM (`ops.gemm_tn32`, csrc/gemm_tn32_sm90.cu) alone at every shape the training step
gives it.  The shapes are recorded, not listed by hand: one eager `TrainStep` at the bench configuration runs with
`ops.gemm_tn32` wrapped, and each distinct call (rows, m, n, strides, prologue modes, column sums) is then timed on
seeded inputs of the same layout with CUDA events, the kernel alone and warm.

    python tools/bench_tn32.py [--tree DIR] [--batch 8] [--npoints 20000] [--windows 5]

--tree: import the package from another checkout of this repository (its library already built), so two builds can be
timed one after the other in the same command.  Prints one JSON line per shape: calls per step, ms per launch (median of
`--windows` windows, with min and max), algorithmic GB/s (fp32 operands read once, the pooled gradient and arg-max
rows, C and the column sums written once) and that rate over the HBM peak (MEASURED_PEAKS.json `hbm_gbs` when present,
else the H100 SXM data sheet's 3.35 TB/s).  A last line gives the card, its power limit and the sum over the step."""
import argparse
import json
import subprocess
import sys
import warnings
from pathlib import Path

import numpy as np
import torch

HBM_GBS = 3350.0


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--tree", default=str(Path(__file__).resolve().parents[1]))
    p.add_argument("--batch", type=int, default=8)
    p.add_argument("--npoints", type=int, default=20000)
    p.add_argument("--windows", type=int, default=5)
    p.add_argument("--window-ms", type=float, default=100.0, help="device time per timing window")
    return p.parse_args()


def record_shapes(a):
    """-> {signature: calls} of ops.gemm_tn32 during one eager training step (after one step of warm-up)."""
    from coda_neurips2023_b200 import ops, synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.engine import TrainStep
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args()
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model = model.cuda().train()
    crit = build_criterion(args, cfg).cuda()
    step = TrainStep(args, model, crit, torch.device("cuda", 0))
    batch = synthetic.to_device(synthetic.make_batch(a.batch, a.npoints, seed=0), "cuda")
    np.random.seed(0)
    step(batch, 0.0)
    torch.cuda.synchronize()

    calls = {}
    inner = ops.gemm_tn32

    def recorder(x, y, *, a_mode=ops.A32_PLAIN, a2=None, group=0, b_mode=ops.A32_PLAIN, out=None, colsum_out=None,
                 **kw):
        rows, m = x.shape
        sig = (rows, m, y.shape[1], x.stride(0), a_mode, a2.stride(0) if a_mode == ops.A32_BN_BWD else 0, group,
               y.stride(0), b_mode, colsum_out is not None)
        calls[sig] = calls.get(sig, 0) + 1
        return inner(x, y, a_mode=a_mode, a2=a2, group=group, b_mode=b_mode, out=out, colsum_out=colsum_out, **kw)

    ops.gemm_tn32 = recorder
    try:
        step(batch, 0.0)
        torch.cuda.synchronize()
    finally:
        ops.gemm_tn32 = inner
    del step, model, crit, batch
    torch.cuda.empty_cache()
    return calls


def case(sig):
    """-> (launch, algorithmic bytes) on seeded inputs with the recorded layout"""
    from coda_neurips2023_b200 import ops

    rows, m, n, lda, a_mode, lda2, group, ldb, b_mode, colsum = sig
    g = torch.Generator(device="cuda").manual_seed(rows + m + n)
    dev = "cuda"
    x = torch.randn(rows, lda, device=dev, generator=g)[:, :m]
    y = torch.randn(rows, ldb, device=dev, generator=g)[:, :n]
    kw = {}
    nbytes = 4.0 * rows * (m + n) + 4.0 * m * n + (4.0 * m if colsum else 0.0)
    if a_mode != ops.A32_PLAIN:
        v = lambda c: torch.rand(c, device=dev, generator=g) + 0.5  # noqa: E731
        kw.update(a_scale=v(m), a_shift=v(m) - 1.0, a_alpha=(v(m) - 1.0) * 0.1, a_beta=(v(m) - 1.0) * 0.1)
    if a_mode == ops.A32_BN_BWD:
        kw["a2"] = torch.randn(rows, lda2, device=dev, generator=g)[:, :m]
        nbytes += 4.0 * rows * m
    elif a_mode in (ops.A32_BN_BWD_POOLED, ops.A32_BN_BWD_POOLED_PRE):
        kw["a2"] = torch.randn(rows // group, m, device=dev, generator=g)
        kw["argmax"] = torch.randint(0, group, (rows // group, m), device=dev, dtype=torch.uint8, generator=g)
        kw["group"] = group
        nbytes += 5.0 * (rows // group) * m
    if b_mode == ops.A32_AFFINE_RELU:
        kw.update(b_mode=b_mode, b_scale=torch.rand(n, device=dev, generator=g) + 0.5,
                  b_shift=torch.randn(n, device=dev, generator=g) * 0.1)
    out = torch.empty(m, n, device=dev)
    cs = torch.empty(m, device=dev) if colsum else None
    return (lambda: ops.gemm_tn32(x, y, a_mode=a_mode, out=out, colsum_out=cs, **kw)), nbytes


def time_windows(fn, windows, window_ms):
    """-> ms per call in each window.  The calls are replayed from a CUDA graph, as in the training step, so the host
    cost of a call (ctypes, tensor-map encoding) is not part of the number for the short launches."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    reps = max(10, int(window_ms / max(e0.elapsed_time(e1), 1e-3)))
    graph, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        for _ in range(reps):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / reps)
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def main():
    a = parse()
    tree = Path(a.tree).resolve()
    sys.path.insert(0, str(tree))
    from coda_neurips2023_b200 import ops

    assert Path(ops.__file__).resolve().is_relative_to(tree), ops.__file__
    assert torch.cuda.is_available(), "bench_tn32 times the kernel on the GPU"
    try:
        peak = float(json.loads((tree / "MEASURED_PEAKS.json").read_text())["hbm_gbs"])
    except (OSError, KeyError, ValueError):
        peak = HBM_GBS
    calls = record_shapes(a)
    names = {ops.A32_PLAIN: "plain", ops.A32_BN_BWD: "bn_bwd", ops.A32_BN_BWD_POOLED: "bn_bwd_pooled",
             ops.A32_BN_BWD_POOLED_PRE: "bn_bwd_pooled_pre", ops.A32_AFFINE_RELU: "affine_relu"}
    step_ms = 0.0
    for sig in sorted(calls, key=lambda s: -s[0] * (s[1] + s[2])):
        rows, m, n, lda, a_mode, lda2, group, ldb, b_mode, colsum = sig
        fn, nbytes = case(sig)
        ts = time_windows(fn, a.windows, a.window_ms)
        ms = float(np.median(ts))
        step_ms += ms * calls[sig]
        gbs = nbytes / (ms * 1e-3) / 1e9
        print(json.dumps({"rows": rows, "m": m, "n": n, "lda": lda, "ldb": ldb, "a_mode": names[a_mode],
                          "b_mode": names[b_mode], "group": group, "colsum": colsum, "calls_per_step": calls[sig],
                          "ms": round(ms, 4), "ms_min": round(min(ts), 4), "ms_max": round(max(ts), 4),
                          "algorithmic_GBps": round(gbs, 1), "hbm_frac": round(gbs / peak, 3)}), flush=True)
        del fn
        torch.cuda.empty_cache()
    print(json.dumps({"tree": str(tree), "card": card(), "hbm_peak_GBps": peak, "shapes": len(calls),
                      "launches_per_step": sum(calls.values()), "tn32_ms_per_step": round(step_ms, 3)}), flush=True)


if __name__ == "__main__":
    main()
