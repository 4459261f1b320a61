#!/usr/bin/env python
"""Benchmark of the CoDA training step (BASELINE.json metric: training scenes/sec on
20 000-point SUN RGB-D-shaped synthetic clouds, 256 queries).

    python bench.py --gpus 1 --steps 10 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port P bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # the reference's CPU path on the host cores

One "step" = H2D of one batch (e2e leg only) + model forward + Hungarian-matched criterion +
backward + single gradient all-reduce + clip + AdamW on `--batch-per-gpu` scenes per GPU.
Prints ONE JSON line (rank 0).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time
import warnings
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

METRIC = "training scenes/sec (20k-pt SUN-RGBD synth, 256 queries)"
UNIT = "scenes/s"
# NVIDIA H100 SXM data sheet (700 W card): dense BF16 tensor rate, HBM3 bandwidth.  Used as the roofline peaks when
# no measured peaks are given; a card with a lower power limit does not reach them.
H100_BF16_TFLOPS = 989.0
H100_HBM_GBS = 3350.0
DUMP_SAMPLE = 1 << 20     # parameter / gradient entries kept by --dump-outputs (fixed seeded sample)


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--impl", default="ours", choices=["ours", "reference"])
    p.add_argument("--batch-per-gpu", type=int, default=8)
    p.add_argument("--npoints", type=int, default=20000)
    p.add_argument("--nqueries", type=int, default=256)
    p.add_argument("--cpu-sample-scenes", type=int, default=1)
    p.add_argument("--no-cpu-baseline", action="store_true")
    p.add_argument("--no-graph", action="store_true", help="run the step eagerly instead of as one CUDA graph")
    p.add_argument("--nsplit", type=int, default=3, help="bf16 planes per fp32 operand on the tensor-core path")
    p.add_argument("--num-classes", type=int, default=46, help="text rows (46: SUN RGB-D prompts; 232: ScanNet-200 set)")
    p.add_argument("--image", default="531x730", help="image height x width (ScanNet shape: 968x1296)")
    p.add_argument("--dump-outputs", metavar="DIR", default=None,
                   help="write what the last timed step computed (loss, loss terms, a fixed sample of the updated "
                        "parameters and of their gradients) as DIR/<name>.npy")
    return p.parse_args()


def image_hw(a):
    h, w = a.image.lower().split("x")
    return int(h), int(w)


def workload_config(a, world):
    h, w = image_hw(a)
    return {"workload": f"CoDA stage-1 train step: PointNet++ SA({a.npoints}->2048) + 3DETR enc3/dec8 + CLIP ViT-B/32 "
                        "alignment (32 crops/scene) + Hungarian losses + clip + AdamW",
            "npoints": a.npoints, "nqueries": a.nqueries, "batch_per_gpu": a.batch_per_gpu,
            "global_batch": a.batch_per_gpu * world, "parallelism": f"dp{world}",
            "weights": "random-init (no checkpoints offline)", "num_text_classes": a.num_classes,
            "image_hw": [h, w],
            "l2": "per-step working set (~2 GB of SA / attention activations) >> 50 MB L2; inputs differ per step"}


# --------------------------------------------------------------------------- clocks
class ClockSampler:
    """nvidia-smi sampling DURING the timed region (profiling recipe's clocks line)."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.gpu, self.rows, self.proc = gpu_index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.gpu)], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self) -> dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm = [float(r[1]) for r in self.rows if len(r) > 8 and r[1].replace(".", "").isdigit()]
        mx = [float(r[2]) for r in self.rows if len(r) > 8 and r[2].replace(".", "").isdigit()]
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            if len(r) > 8:
                for n, v in zip(names, r[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# --------------------------------------------------------------------------- CPU (reference) arm
def cpu_step_rate(a, scenes: int, steps: int, threads: int):
    """The reference's CPU path for this step -- its own PyTorch arithmetic (torch CPU ops), the C
    restatement of the CUDA-only pointnet2 ops and scipy for the assignment (oracle/cpu_step.py) --
    timed on `scenes` scenes for `steps` steps.  Returns scenes/s."""
    sys.path.insert(0, str(ROOT / "oracle"))
    sys.path.insert(0, str(ROOT / "tests"))
    import cpu_step
    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.models import build_model

    torch.set_num_threads(threads)
    h, w = image_hw(a)
    args = synthetic.make_args(nqueries=a.nqueries, test_range_max=a.num_classes, image_size_width=w, image_size_height=h)
    cfg = synthetic.SyntheticDatasetConfig(args)
    with cpu_step.installed():
        torch.manual_seed(0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = build_model(args, cfg)
        model = model.to_device("cpu").float().train()
        model.clip_model.eval()
        criterion = build_criterion(args, cfg)
        opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=args.base_lr,
                                weight_decay=args.weight_decay)
        batch = {k: torch.from_numpy(v)
                 for k, v in synthetic.make_batch(scenes, a.npoints, seed=0, image_hw=image_hw(a)).items()}
        times = []
        for _ in range(steps):
            t0 = time.perf_counter()
            opt.zero_grad()
            out = model(batch, curr_epoch=0)
            loss, _ = criterion(out, batch)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(model.parameters(), args.clip_gradient)
            opt.step()
            times.append(time.perf_counter() - t0)
    return scenes / float(np.median(times)), float(np.median(times))


def run_reference(a):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    threads = min(os.cpu_count() or 1, 32)
    steps = max(1, min(a.steps, 2))
    rate, sec = cpu_step_rate(a, a.cpu_sample_scenes, steps, threads)
    line = {
        "impl": "reference", "metric": METRIC, "value": rate, "unit": UNIT, "n_gpus": a.gpus, "steps": steps,
        "warmup": 1, "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "fp32", "data": "synthetic", "config": workload_config(a, 1) | {"batch_per_gpu": a.cpu_sample_scenes,
                                                                                "global_batch": a.cpu_sample_scenes},
        "cpu_baseline": {"value": rate, "unit": UNIT, "cores": threads, "kind": "port",
                         "sample": f"{a.cpu_sample_scenes} scenes/step x {steps} steps (median), full step "
                                   "incl. CLIP ViT-B/32 on 32 crops/scene; reference PyTorch CPU arithmetic + "
                                   "C restatement of its CUDA-only pointnet2 ops"},
        "e2e": {"value": rate, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "reference_scope": "ONE CPU process on this box's host cores, whatever --gpus says: the CPU path does not shard; "
                           "compare an N-GPU line with this value as is (it is not scaled by N)",
    }
    _emit(line)


# --------------------------------------------------------------------------- our arm
def attention_roofline(a, device):
    """CUDA-event timing of the dominant tensor-core kernel -- the encoder self-attention forward
    (L = 2048 seeds, 4 heads x 64) -- in isolation on the step's shapes; algorithmic FLOPs =
    4 * B * H * Lq * Lk * hd per launch (QK^T + PV)."""
    import ctypes

    from coda_neurips2023_b200 import _lib

    peaks = {}
    try:
        peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
    except OSError:
        pass
    peak = float(peaks.get("bf16_tflops", H100_BF16_TFLOPS))
    b, h, lq, lk, hd = a.batch_per_gpu, 4, 2048, 2048, 64
    q = torch.randn(lq, b, h * hd, device=device)
    k = torch.randn(lk, b, h * hd, device=device)
    v = torch.randn(lk, b, h * hd, device=device)
    L = _lib.lib()
    L.coda_attention_workspace_bytes.restype = ctypes.c_longlong
    from coda_neurips2023_b200 import attention_launch

    ns = attention_launch.FORWARD_NSPLIT      # the split the step's attention forward actually runs on
    ws = torch.empty(int(L.coda_attention_workspace_bytes(b, h, lq, lk, hd, ns)), dtype=torch.uint8, device=device)
    out = torch.empty_like(q)
    lse = torch.empty(b * h, lq, device=device)
    stream = ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check(L.coda_attention_pack(b, h, lq, lk, hd, ns, ctypes.c_float(hd ** -0.5), P(q), P(k), P(v), P(ws),
                                     stream), "attention_pack")

    def launch():
        # dropout 0.1 as in the training step (enc_dropout): the mask is generated inside the kernel
        return L.coda_attention_fwd_packed(b, h, lq, lk, hd, ns, P(ws), P(out), P(lse), ctypes.c_float(0.1), 12345,
                                           None, stream)

    for _ in range(3):
        _lib.check(launch(), "attention_fwd_packed")
    torch.cuda.synchronize()
    reps = 20
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        launch()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    flops = 4.0 * b * h * lq * lk * hd          # algorithmic: QK^T + PV, 2 flops per MAC
    achieved = flops / (ms * 1e-3) / 1e12
    nprod = {1: 1.0, 2: 3.0, 3: 5.5}[ns]       # QK^T: 1 / 3 / 6 plane products, PV: 1 / 3 / 5 (P carries 2 planes)
    return {"bound": "tensor", "kernel": "attn_fwd_kernel<64,%d> (wgmma fused encoder self-attention forward, "
            "L=2048, 4 heads x 64, batch %d)" % (ns, b),
            "achieved": achieved, "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak,
            "peak_source": "MEASURED_PEAKS.json bf16_tflops (burst; kernel timed alone)" if peaks
            else "H100 SXM data sheet, dense BF16",
            "flops_per_launch": flops, "ms_per_launch": ms, "traffic": None,
            "tensor_pipe_flops_per_launch": flops * nprod,
            "tensor_pipe_frac": achieved * nprod / peak,
            "note": "fp32 operands are split into %d bf16 planes, the tensor pipe executes %.1f bf16 MMAs per "
                    "algorithmic MMA; `achieved`/`frac` count algorithmic FLOPs only" % (ns, nprod)}


def _time_launch(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _attn_split():
    from coda_neurips2023_b200 import attention_launch

    return attention_launch.FORWARD_NSPLIT


def _peaks():
    try:
        return json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
    except OSError:
        return {}


def sa_wgrad_roofline(a, device):
    """The weight-gradient kernel (gemm_tn32_kernel<128>, every weight gradient of the step), timed alone on its
    longest launch: the weight gradient of the third set-abstraction
    layer, dW2 (256 x 128) = dY2^T A2 over R = B * 2048 * 64 rows, with the step's prologues (dY2 from the pre-BN
    activation y2 + the max-pooled gradient; A2 = relu(bn(y1))).  The kernel streams both fp32 activations once:
    algorithmic bytes = 4 R (256 + 128) (+ 21 MB pooled gradient / arg-max); peak = MEASURED_PEAKS.json hbm_gbs."""
    from coda_neurips2023_b200 import ops

    peaks = _peaks()
    peak = float(peaks.get("hbm_gbs", H100_HBM_GBS))
    rows, m, n, group = a.batch_per_gpu * 2048 * 64, 256, 128, 64
    y2 = torch.randn(rows, m, device=device)
    y1 = torch.randn(rows, n, device=device)
    dp = torch.randn(rows // group, m, device=device)
    arg = torch.randint(0, group, (rows // group, m), device=device, dtype=torch.uint8)
    v = lambda c: (torch.rand(c, device=device) + 0.5, torch.randn(c, device=device) * 0.1)  # noqa: E731
    (sa, ta), (al, be), (sb, tb) = v(m), v(m), v(n)
    out = torch.empty(m, n, device=device)
    # the step's form: the pooled gradient arrives masked and scaled (coda_bn_relu_bwd_reduce_pooled `dprime`)
    ms = _time_launch(lambda: ops.gemm_tn32(y2, y1, a_mode=ops.A32_BN_BWD_POOLED_PRE, a_scale=sa, a_shift=ta, a_alpha=al,
                                            a_beta=be, a2=dp, argmax=arg, group=group, b_mode=ops.A32_AFFINE_RELU,
                                            b_scale=sb, b_shift=tb, out=out))
    nbytes = 4.0 * rows * (m + n) + 5.0 * (rows // group) * m + 4.0 * m * n
    achieved = nbytes / (ms * 1e-3) / 1e9
    return {"bound": "hbm", "kernel": "gemm_tn32_kernel<128> (wgmma weight-gradient GEMM on fp32 rows, BatchNorm-backward / "
            "BatchNorm+ReLU prologues in-kernel; SA layer 3: dW (%d x %d) over %d rows)" % (m, n, rows),
            "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
            "peak_source": "MEASURED_PEAKS.json hbm_gbs" if peaks else "H100 SXM data sheet, HBM3",
            "bytes_per_launch": nbytes, "ms_per_launch": ms, "traffic": None,
            "useful_tflops": 2.0 * rows * m * n / (ms * 1e-3) / 1e12,
            "note": "working set (1.6 GB) >> 50 MB L2: every timed launch streams from HBM"}


def sa_forward_roofline(a, device):
    """gemm_a32_kernel<3,128,...> on the forward of the same layer: y2 (R x 256) = relu(bn(y1)) W2^T, y1 read as fp32
    with the BatchNorm+ReLU prologue, BatchNorm statistics of y2 produced by the epilogue.  Algorithmic bytes = y1 read
    once + y2 written once."""
    from coda_neurips2023_b200 import ops

    peaks = _peaks()
    peak = float(peaks.get("hbm_gbs", H100_HBM_GBS))
    rows, k, n, ns = a.batch_per_gpu * 2048 * 64, 128, 256, a.nsplit
    y1 = torch.randn(rows, k, device=device)
    wp = ops.pack_split(torch.randn(n, k, device=device) / k ** 0.5, n, k, k, 1, 3)
    sc, sh = torch.rand(k, device=device) + 0.5, torch.randn(k, device=device) * 0.1
    out = torch.empty(rows, n, device=device)
    ms = _time_launch(lambda: ops.gemm_a32(y1, wp, n, mode=ops.A32_AFFINE_RELU, scale=sc, shift=sh, out=out,
                                           want_stats=True, nsplit=ns))
    nbytes = 4.0 * rows * (k + n) + 2.0 * ns * n * k
    achieved = nbytes / (ms * 1e-3) / 1e9
    return {"bound": "hbm", "kernel": "gemm_a32_kernel<%d,128> (wgmma GEMM, fp32 A split in-kernel into register "
            "fragments, BN+ReLU prologue, BN-statistics epilogue; SA layer 3 forward: %d x %d x %d)" % (ns, rows, n, k),
            "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
            "peak_source": "MEASURED_PEAKS.json hbm_gbs" if peaks else "H100 SXM data sheet, HBM3",
            "bytes_per_launch": nbytes, "ms_per_launch": ms, "traffic": None,
            "useful_tflops": 2.0 * rows * n * k / (ms * 1e-3) / 1e12,
            "tensor_pipe_tflops": 2.0 * rows * n * k * {2: 3, 3: 6}[ns] / (ms * 1e-3) / 1e12}


def run_ours(a):
    import torch.distributed as dist

    from coda_neurips2023_b200 import _lib, ops, synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.engine import TrainStep
    from coda_neurips2023_b200.models import build_model

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench.py --impl ours needs a GPU (no CPU fallback)"
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    torch.backends.cudnn.allow_tf32 = False       # fp32 arithmetic, like the parity runs
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True

    h, w = image_hw(a)
    args = synthetic.make_args(nqueries=a.nqueries, batchsize_per_gpu=a.batch_per_gpu, ngpus=world,
                               test_range_max=a.num_classes, image_size_width=w, image_size_height=h)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(rank)  # per-rank seed as the reference (main.py:982-985); TrainStep broadcasts rank 0's state
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model = model.to(device).train()
    criterion = build_criterion(args, cfg).to(device)
    ops.DEFAULT_NSPLIT = a.nsplit
    step = TrainStep(args, model, criterion, device)
    np.random.seed(1000 + rank)

    nb = 4  # distinct batches, cycled; seed = rank-dependent (DistributedSampler-like sharding)
    host = [{k: torch.from_numpy(np.ascontiguousarray(v)).pin_memory()
             for k, v in synthetic.make_batch(a.batch_per_gpu, a.npoints, seed=100 * rank + i,
                                              image_hw=image_hw(a)).items()}
            for i in range(nb)]
    h2d_bytes = sum(t.numel() * t.element_size() for t in host[0].values())
    resident = [step.to_device(h) for h in host]
    torch.cuda.synchronize()
    use_graph = not a.no_graph
    graph_note = None
    if use_graph:
        try:
            step.capture(resident[0])
        except Exception as e:  # noqa: BLE001  (report, run eagerly: the number is still valid, just launch-bound)
            use_graph, step.graph = False, None
            graph_note = f"capture failed: {type(e).__name__}: {str(e)[:160]}"

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms: float) -> float:
        if world == 1:
            return ms
        t = torch.tensor([ms], device=device, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    sampler = ClockSampler(local)
    # ---------------- device-resident leg (value) ----------------
    for i in range(a.warmup):
        step(resident[i % nb], 0.0)
    barrier()
    if rank == 0:
        sampler.start()
    launches0 = _lib.LAUNCHES
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        loss, loss_terms = step(resident[i % nb], 0.0)
    e1.record()
    barrier()
    launches = (_lib.LAUNCHES - launches0) if not use_graph else step.launches_per_step * a.steps
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, loss, loss_terms, step.flat)
    ms_dev = max_over_ranks(e0.elapsed_time(e1))
    assert torch.isfinite(loss).item(), "non-finite loss"
    # ---------------- end-to-end leg (host buffers, H2D + loss read-back inside) ----------------
    feed = (lambda hb: hb) if use_graph else step.to_device  # graph mode: H2D straight into the static buffers
    for i in range(min(a.warmup, 2)):
        step(feed(host[i % nb]), 0.0)
    barrier()
    e0.record()
    d2h = 0
    for i in range(a.steps):
        loss, _ = step(feed(host[i % nb]), 0.0)
        lv = loss.item()  # device -> host read of the step's result, every step
        d2h = 4
    e1.record()
    barrier()
    ms_e2e = max_over_ranks(e0.elapsed_time(e1))
    clocks = sampler.stop() if rank == 0 else None
    # data-parallel sanity: after the same number of all-reduced steps every rank holds the same weights
    param_spread = 0.0
    if world > 1:
        hi, lo = step.flat.flat_param.detach().clone(), step.flat.flat_param.detach().clone()
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        param_spread = float((hi - lo).abs().max().item())

    if rank != 0:
        _finish(world, device)
        return
    scenes = a.batch_per_gpu * world * a.steps
    line = {
        "metric": METRIC, "value": scenes / (ms_dev * 1e-3), "unit": UNIT, "n_gpus": world, "steps": a.steps,
        "warmup": a.warmup, "ms_per_step": ms_dev / a.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "fp32", "data": "synthetic", "config": workload_config(a, world),
        "e2e": {"value": scenes / (ms_e2e * 1e-3), "unit": UNIT, "h2d_bytes_per_step": h2d_bytes,
                "d2h_bytes_per_step": d2h, "ms_per_step": ms_e2e / a.steps},
        "gpu_launches": launches, "gpu_launches_note": "C-ABI kernel-launching calls into libcoda_b200.so inside the "
                                                        "timed region (cuBLAS/cuDNN launches of torch not counted)",
        "clocks": clocks, "final_loss": lv, "cuda_graph": use_graph, "cuda_graph_note": graph_note,
        "operand_split": a.nsplit, "attention_forward_operand_split": _attn_split(),
        "param_spread_across_ranks": param_spread,
        "grad_allreduce_bytes": step.flat.nbytes(),
    }
    line["roofline"] = sa_wgrad_roofline(a, device)
    # the kernels next in line, same measurement method (kernel alone, CUDA events)
    line["roofline_more"] = [sa_forward_roofline(a, device), attention_roofline(a, device)]
    if world == 1 and not a.no_cpu_baseline:
        threads = min(os.cpu_count() or 1, 32)  # more threads only slow these small CPU ops down
        rate, sec = cpu_step_rate(a, 1, 1, threads)
        line["cpu_baseline"] = {"value": rate, "unit": UNIT, "cores": threads, "kind": "port",
                                "sample": f"1 scene, 1 full step ({sec:.1f} s): reference PyTorch CPU arithmetic + "
                                          "C restatement of its CUDA-only ops; use --impl reference for more steps"}
    _emit(line)
    _finish(world, device)


def dump_outputs(out_dir, loss, loss_terms, flat):
    """What the last timed step computed, as float32 / float64 .npy files: the loss, every scalar loss term, and the
    same seeded sample of the updated parameters and of their gradients (the full vectors are larger than needed
    to compare two builds)."""
    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    np.save(d / "loss.npy", np.array([float(loss)], dtype=np.float64))
    for k, v in sorted(loss_terms.items()):
        if isinstance(v, torch.Tensor) and v.numel() == 1:
            np.save(d / f"loss_term.{k}.npy", np.array([float(v.detach())], dtype=np.float64))
    total = flat.flat_param.numel()
    gen = np.random.default_rng(0)
    idx = np.sort(gen.choice(total, size=min(DUMP_SAMPLE, total), replace=False))
    sel = torch.from_numpy(idx).to(flat.flat_param.device)
    np.save(d / "param_sample_index.npy", idx.astype(np.float64))
    np.save(d / "param_sample.npy", flat.flat_param.detach()[sel].float().cpu().numpy())
    np.save(d / "grad_sample.npy", flat.flat_grad.detach()[sel].float().cpu().numpy())


def _finish(world, device):
    """Leave without tearing NCCL down: destroying a communicator that a live CUDA graph still
    references can hang at interpreter exit; every rank is done with collectives here."""
    sys.stdout.flush()
    sys.stderr.flush()
    if world > 1:
        torch.cuda.synchronize(device)
        os._exit(0)


_RESULT_FD = None


def _emit(line: dict) -> None:
    """the ONE JSON line, on the process's real stdout"""
    text = json.dumps(line) + "\n"
    if _RESULT_FD is None:
        sys.stdout.write(text)
        sys.stdout.flush()
    else:
        os.write(_RESULT_FD, text.encode())


def main():
    global _RESULT_FD
    a = parse()
    # stdout carries the result line and nothing else: native libraries print there too (NCCL's
    # "NCCL version ..." banner under NCCL_DEBUG=VERSION), so file descriptor 1 is pointed at stderr for the
    # duration of the run and the result is written to a private duplicate of the original descriptor
    sys.stdout.flush()
    try:
        _RESULT_FD = os.dup(1)
        os.dup2(2, 1)
    except OSError:          # no usable stderr / stdout descriptors: print the line the plain way
        _RESULT_FD = None
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)


if __name__ == "__main__":
    main()
