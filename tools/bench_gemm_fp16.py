"""Time the CLIP tower's fp16 GEMMs (ViT-B/32 on 256 crops) with the epilogue each one uses, beside cuBLAS
(`F.linear`, no fused epilogue) on the same operands.  Prints one JSON line per shape and build: ms, TFLOP/s and the
fraction of the H100 SXM's 989 TFLOP/s dense-fp16 data-sheet rate.

    python tools/bench_gemm_fp16.py [--roots TREE [TREE ...]] [--rounds R]

With several source trees (each with its library built), the trees run in turn, R rounds, each in a process of its own,
so that two builds are compared in one command under the same conditions.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

PEAK_TFLOPS = 989.0
# name, m, n, k, bias, act (2 = QuickGELU), residual
SHAPES = [("qkv", 12800, 2304, 768, True, 0, False),
          ("out_proj", 12800, 768, 768, True, 0, True),
          ("c_fc", 12800, 3072, 768, True, 2, False),
          ("c_proj", 12800, 768, 3072, True, 0, True),
          ("patch", 12544, 768, 3072, False, 0, False),
          ("project", 12800, 512, 768, False, 0, False)]


def timeit(fn, reps=50, warm=10):
    import torch

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


def worker(root: Path):
    sys.path.insert(0, str(root.resolve()))
    import torch
    from coda_neurips2023_b200 import ops

    assert torch.cuda.is_available(), "needs a CUDA device"
    for name, m, n, k, bias, act, res in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(0)
        a = (torch.randn(1, 1, m, k, device="cuda", generator=g) * 0.5).half()
        b = (torch.randn(1, 1, n, k, device="cuda", generator=g) * k ** -0.5).half()
        bv = torch.randn(n, device="cuda", generator=g) if bias else None
        r = torch.randn(m, n, device="cuda", generator=g).half() if res else None
        out = torch.empty(1, m, n, device="cuda", dtype=torch.float16)
        ms = timeit(lambda: ops.gemm_nt(a, b, m, n, bias=bv, act=act, out=out, residual=r))
        a2, b2 = a[0, 0], b[0, 0]
        cublas = timeit(lambda: torch.nn.functional.linear(a2, b2))
        tf = 2.0 * m * n * k / ms / 1e9
        print(json.dumps({"tree": str(root), "shape": name, "m": m, "n": n, "k": k, "ms": round(ms, 4),
                          "tflops": round(tf, 1), "frac_peak": round(tf / PEAK_TFLOPS, 3),
                          "cublas_ms": round(cublas, 4),
                          "cublas_tflops": round(2.0 * m * n * k / cublas / 1e9, 1)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--roots", type=Path, nargs="+", default=[Path(__file__).resolve().parents[1]])
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--worker", type=Path, default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.worker)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None}),
          flush=True)
    for _ in range(args.rounds):
        for root in args.roots:
            subprocess.run([sys.executable, __file__, "--worker", str(root)], check=True)


if __name__ == "__main__":
    main()
