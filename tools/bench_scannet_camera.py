"""SUN RGB-D camera vs ScanNet camera at the ScanNet stage-1 configuration (scripts/coda_scannet_stage1.sh: 8 scenes per
GPU x 40 000 points, 1296 x 968 images, 128 queries, 10 seen / 60 prompts), in one process, alternating the two:

  * the whole training step (captured CUDA graph), CUDA events around `--steps` steps, `--rounds` alternations;
  * ops.boxes_in_image alone (B = 8, Q = 128 and 256): 100 calls captured in a CUDA graph, CUDA events around
    `--launches` calls.

Prints one line per measurement and a JSON summary with the card's name and power limit.

    python tools/bench_scannet_camera.py [--steps 20] [--rounds 5] [--launches 2000] [--out result.json]
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
from coda_neurips2023_b200 import ops, synthetic  # noqa: E402
from coda_neurips2023_b200.criterion import build_criterion  # noqa: E402
from coda_neurips2023_b200.engine import TrainStep  # noqa: E402
from coda_neurips2023_b200.models import build_model  # noqa: E402

STAGE1 = dict(nqueries=128, train_range_max=10, test_range_max=60, image_size_width=1296, image_size_height=968,
              matcher_giou_cost=2.0, matcher_center_cost=0.0, matcher_objectness_cost=0.0, loss_no_object_weight=0.25,
              base_lr=1.4142e-4)
DATASET = {"sunrgbd": "sunrgbd_anonymous_aligned_image", "scannet": "scannet_anonymous_aligned_image"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def make_step(camera, batch, npoints):
    args = synthetic.make_args(dataset_name=DATASET[camera], **STAGE1)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model = model.cuda().train()
    step = TrainStep(args, model, build_criterion(args, cfg).cuda(), torch.device("cuda", 0))
    data = synthetic.to_device(synthetic.make_batch(batch, npoints, seed=0, image_hw=(968, 1296), camera=camera), "cuda")
    np.random.seed(0)
    step.capture(data, warmup=3)
    for _ in range(3):
        step(data, 0.0)
    torch.cuda.synchronize()
    return step, data


def time_steps(step, data, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        loss, _ = step(data, 0.0)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, float(loss)


def time_projection(camera, b, q, launches):
    data = synthetic.to_device(synthetic.make_batch(b, 2000, seed=1, image_hw=(968, 1296), camera=camera), "cuda")
    gen = torch.Generator(device="cuda").manual_seed(0)
    corners = torch.rand(b, q, 8, 3, device="cuda", generator=gen) * 4 - 2
    size = torch.rand(b, q, 3, device="cuda", generator=gen) + 0.1
    for _ in range(20):
        ops.boxes_in_image(corners, size, data, camera=camera)
    torch.cuda.synchronize()
    # 100 calls captured in one CUDA graph: the replay times the device work, not the host's enqueue rate
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(100):
            ops.boxes_in_image(corners, size, data, camera=camera)
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = max(launches // 100, 1)
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (reps * 100) * 1e3     # us per call on the device (operand casts + the kernel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--npoints", type=int, default=40000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scannet_camera: needs a CUDA device")
    gpu = card()
    print("card:", gpu, flush=True)
    res = {"card": gpu, "batch": a.batch, "npoints": a.npoints, "step_ms": {"sunrgbd": [], "scannet": []},
           "boxes_in_image_us": {"sunrgbd": {}, "scannet": {}}}
    steps = {cam: make_step(cam, a.batch, a.npoints) for cam in ("sunrgbd", "scannet")}
    for r in range(a.rounds):
        for cam in ("sunrgbd", "scannet"):
            ms, loss = time_steps(*steps[cam], a.steps)
            res["step_ms"][cam].append(round(ms, 3))
            print(f"round {r} {cam:8s} step {ms:8.3f} ms  (loss {loss:.4f})", flush=True)
    for q in (128, 256):
        for r in range(3):
            for cam in ("sunrgbd", "scannet"):
                us = time_projection(cam, a.batch, q, a.launches)
                res["boxes_in_image_us"][cam].setdefault(str(q), []).append(round(us, 2))
                print(f"boxes_in_image B={a.batch} Q={q} {cam:8s} {us:7.2f} us/call", flush=True)
    for cam in ("sunrgbd", "scannet"):
        t = res["step_ms"][cam]
        print(f"{cam:8s} step median {np.median(t):.3f} ms, min {min(t):.3f}, max {max(t):.3f}")
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
