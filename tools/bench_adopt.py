"""Cost of TrainStep(optimizer=AdamW) at bench.py's shape (8 scenes x 20 000 points, 256 queries): launches per
captured step and step time with and without an adopted optimizer (alternating rounds in one process), and the time
of one save_checkpoint (model + optimizer state_dict through torch.save; the moments are read from the device then).
    python tools/bench_adopt.py --out DIR"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import warnings
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from coda_neurips2023_b200 import synthetic  # noqa: E402
from coda_neurips2023_b200.criterion import build_criterion  # noqa: E402
from coda_neurips2023_b200.engine import TrainStep, _no_decay  # noqa: E402
from coda_neurips2023_b200.models import build_model  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def adamw(args, model):
    """the reference's build_optimizer"""
    decay, no_decay = [], []
    for name, p in model.named_parameters():
        if p.requires_grad:
            (no_decay if args.filter_biases_wd and _no_decay(name, p) else decay).append(p)
    groups = ([{"params": no_decay, "weight_decay": 0.0}] if args.filter_biases_wd else []) + \
        [{"params": decay, "weight_decay": args.weight_decay}]
    return torch.optim.AdamW(groups, lr=args.base_lr)


def save_checkpoint(path, model, opt):
    torch.save({"model": model.state_dict(), "optimizer": opt.state_dict(), "epoch": 0, "args": None,
                "best_val_metrics": {}}, path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_adopt: needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    args = synthetic.make_args()
    cfg = synthetic.SyntheticDatasetConfig(args)
    data = synthetic.to_device(synthetic.make_batch(8, 20000, seed=0), "cuda")
    tmp = tempfile.mkdtemp(prefix="coda_bench_adopt_")

    def make(optimizer_from=None):
        torch.manual_seed(0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = build_model(args, cfg)
        model = model.cuda().train()
        opt = None
        if optimizer_from is not None:
            opt = adamw(args, model)
            sd = torch.load(optimizer_from, map_location="cpu", weights_only=False)
            model.load_state_dict(sd["model"])
            opt.load_state_dict(sd["optimizer"])
        step = TrainStep(args, model, build_criterion(args, cfg).cuda(), dev, optimizer=opt)
        np.random.seed(0)
        step.capture(data, warmup=3)
        for _ in range(3):
            step(data, 0.0)
        torch.cuda.synchronize()
        return step, model, opt

    gpu = card()
    print("card:", gpu, flush=True)
    plain = make()
    # a loaded state to adopt (the moments' values do not change the step's work)
    ckpt = os.path.join(tmp, "seed.pth")
    seed_model = plain[1]
    seed_opt = adamw(args, seed_model)
    for grp in seed_opt.param_groups:
        for p in grp["params"]:
            seed_opt.state[p] = {"step": torch.tensor(3.0), "exp_avg": torch.full_like(p, 1e-4),
                                 "exp_avg_sq": torch.full_like(p, 1e-8)}
    save_checkpoint(ckpt, seed_model, seed_opt)
    del seed_opt
    adopted = make(optimizer_from=ckpt)
    made = {"plain": plain[0], "adopted": adopted[0]}
    res = {"card": gpu, "launches_per_step": {k: s.launches_per_step for k, s in made.items()},
           "ms": {k: [] for k in made}}
    for r in range(a.rounds):
        for name, step in made.items():
            ms = timed(lambda: step(data, 0.0), a.steps)
            res["ms"][name].append(round(ms, 3))
            print(f"round {r} {name:8s} {ms:8.3f} ms/step", flush=True)
    for name in made:
        t = res["ms"][name]
        print(f"{name:8s} median {np.median(t):.3f} ms, min {min(t):.3f}, max {max(t):.3f}; "
              f"launches_per_step {res['launches_per_step'][name]}", flush=True)
    # save_checkpoint of the adopted run, three calls, each timed and reported
    _, model, opt = adopted
    path = os.path.join(tmp, "checkpoint.pth")
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        save_checkpoint(path, model, opt)
        times.append(round((time.perf_counter() - t0) * 1e3, 1))
    res["save_checkpoint_ms"] = times
    res["checkpoint_bytes"] = os.path.getsize(path)
    res["moment_bytes"] = 2 * adopted[0].optimizer.exp_avg.numel() * 4
    print(f"save_checkpoint {times} ms, file {res['checkpoint_bytes'] / 1e6:.1f} MB, "
          f"moments {res['moment_bytes'] / 1e6:.1f} MB", flush=True)
    for f in os.listdir(tmp):
        os.remove(os.path.join(tmp, f))
    os.rmdir(tmp)
    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "bench_adopt.json").write_text(json.dumps(res, indent=1) + "\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
