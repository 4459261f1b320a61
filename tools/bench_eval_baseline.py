"""The 3DETR + CLIP baseline's test-time evaluation on one GPU (`--model_name 3detrmulticlasshead --if_with_clip
--test_only`), at the batch of test_release_models.sh: 48 synthetic SUN RGB-D scenes x 20 000 points, 128 queries,
730 x 531 images, a random-init ViT-B/16 (the tower's real 197-token geometry), 46 classes; then the ScanNet shape
(1296 x 968 images, 60 classes) once.

    python tools/bench_eval_baseline.py [--reps N] [--cmp]

Prints JSON lines: the card (name, power limit, max SM clock); per shape the eval forward with and without the
classification step (CUDA events, median), the usable crops per batch, the crop + tower + classify time alone, the
tower's algorithmic TFLOP/s (FLOPs from the shapes below) and the peak allocated memory.  With --cmp, per shape instead
the eval forward of the comparison-class evaluation (if_cmp_class: 20 / 19 classes) and of the real-test one on the same
model and batch, alternated (CUDA events, median of N each)."""
import argparse
import json
import subprocess
import sys
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from coda_neurips2023_b200 import synthetic  # noqa: E402
from coda_neurips2023_b200.models import build_model  # noqa: E402
from param_fill import fill_by_name  # noqa: E402
from running_stats_fill import fill_running_stats_by_name  # noqa: E402

SCENES, POINTS, QUERIES = 48, 20000, 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[torch.cuda.current_device()].split(",")]
    return {"card": name, "power_limit": power, "max_sm_clock": clock}


def vit_flops_per_crop(width=768, layers=12, tokens=197, patch=16, res=224, out_dim=512):
    """Multiply-adds x 2 of one ViT image through the tower: patch embedding, per layer QKV / attention / output
    projection / MLP (4 x width), and the final projection."""
    patches = (res // patch) ** 2
    embed = patches * (3 * patch * patch) * width
    per_layer = tokens * (3 * width * width + width * width + 2 * width * 4 * width) + 2 * tokens * tokens * width
    return 2.0 * (embed + layers * per_layer + width * out_dim)


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return median(ts)


def setup(shape):
    """The model (weights filled by name) and batch of a shape."""
    if shape == "sunrgbd":
        over, hw, camera = dict(dataset_name="sunrgbd_image", test_range_max=46), (531, 730), "sunrgbd"
    else:
        over = dict(dataset_name="scannet50_image", test_range_max=60, image_size_width=1296, image_size_height=968)
        hw, camera = (968, 1296), "scannet"
    args = synthetic.make_args(model_name="3detrmulticlasshead", nqueries=QUERIES, clip_arch="ViT-B/16", **over)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    fill_by_name(model, seed=3)           # geometry heads only matter for how many boxes land in the image
    fill_running_stats_by_name(model, seed=7)
    model.to_device("cuda")
    model.eval()
    batch = synthetic.to_device(synthetic.make_batch(SCENES, POINTS, seed=0, image_hw=hw, camera=camera), "cuda")
    return args, model, batch, hw


def bench(shape, reps):
    args, model, batch, hw = setup(shape)
    with torch.no_grad():
        def with_cls():
            return model(batch, if_real_test=True)

        def without_cls():
            return model(batch, if_test=True)

        out = with_cls()["outputs"]
        without_cls()
        usable = int(out["clip_usable_mask"].sum())
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t_with, t_without = [], []
        for _ in range(reps):           # alternated
            t_with.append(timed(with_cls, 1))
            t_without.append(timed(without_cls, 1))
        peak = torch.cuda.max_memory_allocated()
        t_cls = timed(lambda: model.classify_boxes(batch, dict(out)), reps)
    flops = usable * vit_flops_per_crop()
    return {"shape": shape, "scenes": SCENES, "points": POINTS, "queries": QUERIES, "image_hw": list(hw),
            "classes": args.test_range_max, "crops_per_tower_call": model.CROPS_PER_CALL,
            "eval_forward_ms": round(median(t_with), 2), "eval_forward_without_classification_ms":
            round(median(t_without), 2), "usable_crops": usable, "crop_tower_classify_ms": round(t_cls, 2),
            "tower_alg_gflop": round(flops / 1e9, 1), "tower_alg_tflops": round(flops / t_cls / 1e9, 1),
            "peak_allocated_gib": round(peak / 2 ** 30, 2)}


def bench_cmp(shape, reps):
    """The comparison-class pass (forward(if_cmp_class=True): 20 SUN RGB-D / 19 ScanNet classes) next to the real-test
    pass (46 / 60 classes) on the same model and batch, alternated.  Both crop and encode the same boxes; only the
    text matrix of the classify kernel differs."""
    _, model, batch, hw = setup(shape)
    with torch.no_grad():
        def real_test():
            return model(batch, if_real_test=True)

        def cmp_class():
            return model(batch, if_cmp_class=True)

        real, cmp = real_test()["outputs"], cmp_class()["outputs"]
        t_real, t_cmp = [], []
        for i in range(reps):           # alternated, each pass first in every other round
            if i % 2:
                t_cmp.append(timed(cmp_class, 1))
            t_real.append(timed(real_test, 1))
            if not i % 2:
                t_cmp.append(timed(cmp_class, 1))
    return {"shape": shape, "scenes": SCENES, "points": POINTS, "queries": QUERIES, "image_hw": list(hw),
            "usable_crops": int(cmp["clip_usable_mask"].sum()), "real_test_classes": real["sem_cls_prob"].shape[-1],
            "cmp_classes": cmp["sem_cls_prob"].shape[-1], "real_test_eval_forward_ms": round(median(t_real), 2),
            "cmp_eval_forward_ms": round(median(t_cmp), 2), "reps": reps}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--cmp", action="store_true",
                   help="time the comparison-class pass (if_cmp_class) next to the real-test pass instead")
    a = p.parse_args()
    print(json.dumps(card()), flush=True)
    if a.cmp:
        print(json.dumps(bench_cmp("sunrgbd", a.reps)), flush=True)
        print(json.dumps(bench_cmp("scannet", a.reps)), flush=True)
        return
    print(json.dumps(bench("sunrgbd", a.reps)), flush=True)
    print(json.dumps(bench("scannet", 2)), flush=True)


if __name__ == "__main__":
    main()
