"""The ViT-B/16 CLIP tower (197 tokens per crop) on its fused fp16 attention, against the route it replaces (pack into
two bf16 planes, the fp32 attention kernel, a cast back to fp16), in one process:

  1. attention alone, L = 197, N = 256 crops, H = 12: the two routes alternated, CUDA events around `--calls` calls
     after a warm-up; the algorithmic bytes (q, k, v read once, fp16 output written once) and FLOPs (4 N H L^2 64)
     against the H100 SXM data sheet's 3.35 TB/s and 989 TFLOP/s;
  2. the tower alone, 256 crops, fp16: new route vs old, alternated (the old one by patching
     attention_launch.forward_half itself), and the two outputs held to the golden's bar against each other;
  3. the training step at the bench shape (8 x 20 000 points, 256 queries, 32 crops per scene), B/16 vs B/32, each a
     captured CUDA graph, `--rounds` alternations of `--steps` steps.

Prints the card (name, power limit, max SM clock) and one line per measurement; writes result.json into --out.

    python tools/bench_clip_b16.py --out OUT_DIR [--calls 50] [--rounds 5] [--steps 20]
"""
import argparse
import json
import subprocess
import sys
import warnings
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from coda_neurips2023_b200 import attention_launch, synthetic  # noqa: E402
from coda_neurips2023_b200.clip import model as cm  # noqa: E402
from coda_neurips2023_b200.criterion import build_criterion  # noqa: E402
from coda_neurips2023_b200.engine import TrainStep  # noqa: E402
from coda_neurips2023_b200.models import build_model  # noqa: E402

HBM_BPS, TC_FLOPS = 3.35e12, 989e12        # H100 SXM data sheet: HBM3 bandwidth, dense fp16 tensor rate


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def old_route(q, k, v, nhead):
    """what _PackedSelfAttention ran for sequences longer than 64 tokens before the resident kernel"""
    return attention_launch.forward(q, k, v, nhead, nsplit=2, half_out=True)[0].to(q.dtype)


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def bench_attention(calls, rounds):
    l, n, h = 197, 256, 12
    e = h * 64
    torch.manual_seed(0)
    q, k, v = (torch.randn(l, n, 3 * e, device="cuda") * 0.8).half().split(e, dim=-1)
    routes = {"resident": lambda: attention_launch.forward_half(q, k, v, h), "bf16_route": lambda: old_route(q, k, v, h)}
    for f in routes.values():
        for _ in range(10):
            f()
    torch.cuda.synchronize()
    a, b = routes["resident"](), routes["bf16_route"]()
    diff = ((a.float() - b.float()).abs().max() / b.float().abs().max()).item()
    bytes_ = 3 * l * n * e * 2 + l * n * e * 2
    flops = 4.0 * n * h * l * l * 64
    bound_us = max(bytes_ / HBM_BPS, flops / TC_FLOPS) * 1e6
    res = {"bytes": bytes_, "flops": flops, "bound_us": round(bound_us, 1), "max_rel_diff": diff,
           "us": {r: [] for r in routes}}
    for _ in range(rounds):
        for name, f in routes.items():
            res["us"][name].append(round(timed(f, calls) * 1e3, 1))
    for name in routes:
        t = float(np.median(res["us"][name]))
        print(f"attention L={l} N={n} H={h} {name:10s} median {t:8.1f} us  ({bytes_ / t / 1e6:.2f} TB/s algorithmic, "
              f"{bound_us / t:.2f} of the HBM bound {bound_us:.1f} us)  rounds {res['us'][name]}", flush=True)
    print(f"attention: {bytes_ / 1e6:.1f} MB, {flops / 1e9:.1f} GFLOP; routes differ by max-rel {diff:.2e}", flush=True)
    return res


def bench_tower(calls, rounds):
    vit = cm.load(None, device="cuda", arch="ViT-B/16").visual
    g = torch.Generator().manual_seed(77)
    x = torch.randn(256, 3, 224, 224, generator=g).half().cuda()
    new_fn = attention_launch.forward_half

    def old_fn(q, k, v, nhead):
        return old_route(q, k, v, nhead) if q.shape[0] > 64 else new_fn(q, k, v, nhead)

    def run(fn):
        attention_launch.forward_half = fn
        try:
            with torch.no_grad():
                return vit(x)[0]
        finally:
            attention_launch.forward_half = new_fn

    routes = {"resident": lambda: run(new_fn), "bf16_route": lambda: run(old_fn)}
    outs = {}
    for name, f in routes.items():
        for _ in range(2):
            outs[name] = f().float()
    torch.cuda.synchronize()
    a, b = outs["resident"], outs["bf16_route"]
    rel = ((a - b).abs().max() / b.abs().max()).item()
    cos = torch.nn.functional.cosine_similarity(a, b, dim=1).min().item()
    res = {"max_rel_diff": rel, "min_cosine": cos, "ms": {r: [] for r in routes}}
    for _ in range(rounds):
        for name, f in routes.items():
            res["ms"][name].append(round(timed(f, calls), 3))
    for name in routes:
        print(f"tower B/16 256 crops {name:10s} median {np.median(res['ms'][name]):8.3f} ms  rounds {res['ms'][name]}",
              flush=True)
    print(f"tower: routes differ by max-rel {rel:.2e}, min cosine {cos:.7f}", flush=True)
    assert rel <= 4e-3 and cos >= 0.99999, "the two routes disagree beyond the golden's bar"
    return res


def make_step(arch):
    args = synthetic.make_args(clip_arch=arch)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model = model.cuda().train()
    step = TrainStep(args, model, build_criterion(args, cfg).cuda(), torch.device("cuda", 0))
    data = synthetic.to_device(synthetic.make_batch(8, 20000, seed=0), "cuda")
    np.random.seed(0)
    step.capture(data, warmup=3)
    for _ in range(3):
        step(data, 0.0)
    torch.cuda.synchronize()
    return step, data


def bench_step(steps, rounds):
    res = {"ms": {"ViT-B/16": [], "ViT-B/32": []}, "loss": {}}
    made = {arch: make_step(arch) for arch in res["ms"]}
    for r in range(rounds):
        for arch, (step, data) in made.items():
            ms = timed(lambda: step(data, 0.0), steps)
            res["ms"][arch].append(round(ms, 3))
            res["loss"][arch] = float(step(data, 0.0)[0])
            print(f"round {r} step {arch} {ms:8.3f} ms  (loss {res['loss'][arch]:.4f})", flush=True)
    for arch in made:
        t = res["ms"][arch]
        print(f"step {arch} median {np.median(t):.3f} ms, min {min(t):.3f}, max {max(t):.3f}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip_b16: needs a CUDA device")
    gpu = card()
    print("card:", gpu, flush=True)
    res = {"card": gpu, "attention": bench_attention(a.calls, a.rounds), "tower": bench_tower(max(a.calls // 10, 3),
                                                                                              a.rounds),
           "step": bench_step(a.steps, a.rounds)}
    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "result.json").write_text(json.dumps(res, indent=1) + "\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
