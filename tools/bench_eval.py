"""Eval-mode inference on one GPU: the pre-encoder's inference kernel (sa_mlp.shared_mlp_max_infer) against the
module-by-module path it replaces, alone and inside the whole eval forward.

    python tools/bench_eval.py [--reps N]

Prints JSON lines: the card (name, power limit, max SM clock); the fused call and the module path at
48 scenes x 2048 seeds x 64 neighbours (CUDA events, the two alternated, median), with the algorithmic bytes /
FLOPs, the tensor-pipe FLOPs the kernel issues (bf16 plane products) and its share of the bound that applies; then
the whole eval forward (model.eval(), no_grad, if_real_test=True, 48 scenes of 20 000 points, 128 queries) with the
kernel and with the module path: ms per batch, scenes/s and peak allocated memory."""
import argparse
import json
import subprocess
import sys
import warnings
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from coda_neurips2023_b200 import ops, sa_mlp, synthetic  # noqa: E402
from coda_neurips2023_b200.pointnet2 import pytorch_utils as pt_utils  # noqa: E402
from param_fill import fill_by_name  # noqa: E402
from running_stats_fill import fill_running_stats_by_name  # noqa: E402

SCENES, SEEDS, GROUP, C0 = 48, 2048, 64, 3
WIDTHS = (C0, 64, 128, 256)
PEAK_BF16 = 989e12          # H100 SXM data sheet, dense
PEAK_HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[torch.cuda.current_device()].split(",")]
    return {"card": name, "power_limit": power, "max_sm_clock": clock}


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def bench_node(reps):
    torch.manual_seed(0)
    mlp = pt_utils.SharedMLP(list(WIDTHS), bn=True).cuda().eval()
    fill_running_stats_by_name(mlp, seed=7)
    for p in mlp.parameters():
        p.requires_grad_(False)
    x = torch.rand((SCENES, C0, SEEDS, GROUP), device="cuda") * 2 - 1

    def fused():
        return mlp.forward_max_pooled_infer(x)

    def module():
        feats = mlp(x)
        return F.max_pool2d(feats, kernel_size=[1, GROUP]).squeeze(-1)

    # the module path's first linear (K = 3) packs its input rows into the per-step activation-plane cache
    # (ops._packed_rows, 2.4 GB here), which only a training step's end clears: clear it after every call
    with torch.no_grad():
        a, b = fused(), module()
        ops._ACT_CACHE.clear()
        dev = ((a - b).abs().max() / b.abs().max()).item()
        del a, b
        for _ in range(2):
            fused(), module()
            ops._ACT_CACHE.clear()
        torch.cuda.synchronize()
        tf, tm = [], []
        for _ in range(reps):
            tf.append(event_ms(fused))
            tm.append(event_ms(module))
            ops._ACT_CACHE.clear()
    rows = SCENES * SEEDS * GROUP
    macs = WIDTHS[0] * WIDTHS[1] + WIDTHS[1] * WIDTHS[2] + WIDTHS[2] * WIDTHS[3]
    flops = 2.0 * rows * macs
    tensor_flops = 2.0 * rows * (6 * WIDTHS[1] * WIDTHS[2] + 5 * WIDTHS[2] * WIDTHS[3])   # plane products issued
    nbytes = 4.0 * (rows * C0 + SCENES * SEEDS * WIDTHS[3])
    t_fused, t_module = median(tf), median(tm)
    bound_tensor, bound_hbm = tensor_flops / PEAK_BF16, nbytes / PEAK_HBM
    bound = max(bound_tensor, bound_hbm)
    return {"what": "sa_mlp_max node, 48 x 2048 x 64", "fused_ms": round(t_fused, 3), "module_ms": round(t_module, 3),
            "speedup": round(t_module / t_fused, 2), "fused_vs_module_max_rel_dev": dev,
            "alg_gflop": round(flops / 1e9, 1), "alg_mb": round(nbytes / 1e6, 1),
            "tensor_pipe_gflop_issued": round(tensor_flops / 1e9, 1),
            "bound": "tensor pipe (bf16 data-sheet peak)" if bound_tensor >= bound_hbm else "HBM",
            "bound_ms": round(bound * 1e3, 3), "fused_share_of_bound": round(bound * 1e3 / t_fused, 3),
            "fused_alg_tflops": round(flops / t_fused / 1e9, 1)}


def bench_forward(reps):
    args = synthetic.make_args(nqueries=128)
    cfg = synthetic.SyntheticDatasetConfig(args)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from coda_neurips2023_b200.models import build_model

        model, _ = build_model(args, cfg)
    fill_by_name(model, seed=3)
    fill_running_stats_by_name(model, seed=7)
    model = model.cuda().eval()
    batch = synthetic.to_device(synthetic.make_batch(SCENES, 20000, seed=0), "cuda")
    real = sa_mlp.infer_applicable

    def run(fused):
        sa_mlp.infer_applicable = real if fused else (lambda *a: False)
        try:
            with torch.no_grad():
                model(batch, if_real_test=True)
        finally:
            sa_mlp.infer_applicable = real
            ops._ACT_CACHE.clear()        # see bench_node

    res = {}
    for fused in (True, False):       # warm-up, then peak memory of one forward each
        run(fused)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        run(fused)
        torch.cuda.synchronize()
        res[fused] = {"peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2), "ms": []}
    for _ in range(reps):
        for fused in (True, False):
            res[fused]["ms"].append(event_ms(lambda: run(fused)))
    out = {"what": f"eval forward, {SCENES} scenes x 20000 points, 128 queries"}
    for fused, tag in ((True, "fused"), (False, "module")):
        ms = median(res[fused]["ms"])
        out[f"{tag}_ms_per_batch"] = round(ms, 2)
        out[f"{tag}_scenes_per_s"] = round(SCENES / ms * 1e3, 1)
        out[f"{tag}_peak_gb"] = res[fused]["peak_gb"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps(card()), flush=True)
    print(json.dumps(bench_node(a.reps)), flush=True)
    print(json.dumps(bench_forward(max(a.reps // 4, 3))), flush=True)


if __name__ == "__main__":
    main()
