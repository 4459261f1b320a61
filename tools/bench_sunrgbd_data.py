"""Device time of one SUN RGB-D stage-1 training batch built by DeviceSunrgbdAugmentor.batch (8 scenes of 50 000 float64
raw points, 531 x 730 canvas, 20 000 samples), CUDA events, median over runs alternated with the numpy restatement
tests/sunrgbd_item_ref.py sunrgbd_item (single thread, per scene -- the CPU restatement, not the reference's code).

    python tools/bench_sunrgbd_data.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

os.environ.setdefault("OMP_NUM_THREADS", "1")
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "oracle"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import sunrgbd_item_ref  # noqa: E402
from coda_neurips2023_b200.datasets import DeviceSunrgbdAugmentor, draw_augmentation_sunrgbd  # noqa: E402
from test_sunrgbd_data_gpu import _big_scenes  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sunrgbd_data: needs a GPU")
    scenes = _big_scenes(8, 1)
    aug = DeviceSunrgbdAugmentor(0, 10, 256)
    gmax = max(len(s[1]) for s in scenes)
    pts, boxes = np.stack([s[0] for s in scenes]), np.zeros((8, gmax, 8))
    for i, s in enumerate(scenes):
        boxes[i, :len(s[1])] = s[1]
    pts, boxes = torch.from_numpy(pts).cuda(), torch.from_numpy(boxes).cuda()          # resident, as in HBM
    npts = [pts.shape[1]] * 8
    nbox = torch.tensor([len(s[1]) for s in scenes], dtype=torch.int32).cuda()
    frames = [torch.from_numpy(s[2]).cuda() for s in scenes]
    K, Rtilt = np.stack([s[3] for s in scenes]), np.stack([s[4] for s in scenes])
    rng = np.random.default_rng(0)
    dev_ms, cpu_ms = [], []
    for r in range(a.reps + 2):
        draws = draw_augmentation_sunrgbd(rng, 8)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        aug.batch(pts, npts, boxes, nbox, frames, K, Rtilt, draws)
        e1.record()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s = scenes[r % 8]
        sunrgbd_item_ref.sunrgbd_item(*s, draws, r % 8, (0, 10), (730, 531), 256)
        t1 = time.perf_counter()
        if r >= 2:
            dev_ms.append(e0.elapsed_time(e1))
            cpu_ms.append((t1 - t0) * 1e3)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"stage1_device_batch8_ms_median": float(np.median(dev_ms)),
                      "stage1_device_batch8_ms_min": float(min(dev_ms)),
                      "restatement_numpy_per_scene_ms_median": float(np.median(cpu_ms)), "reps": a.reps,
                      "gpu": gpu, "note": "raw scenes and frames resident on the device; the draws are uploaded "
                                          "inside the timed window"}))


if __name__ == "__main__":
    main()
