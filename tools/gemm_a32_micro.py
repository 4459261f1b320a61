"""Micro-benchmark of the fp32-A wgmma GEMMs (CUDA events, kernel alone, warm) on the step's shapes.
Prints one JSON line per case: ms, useful TFLOP/s, algorithmic GB/s."""
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from coda_neurips2023_b200 import ops  # noqa: E402


def timeit(fn, reps=20, warm=3):
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


def main():
    only = sys.argv[sys.argv.index("--only") + 1] if "--only" in sys.argv else None   # substring of a case name
    torch.manual_seed(0)
    cases = [("linear 16384x512x512 ns3", 16384, 512, 512, 3, False, False),
             ("linear 2048x512x512 ns3", 2048, 512, 512, 3, False, False),
             ("SA layer2 1Mx128x64 ns3 bn+relu prologue, stats epilogue", 1 << 20, 128, 64, 3, True, False),
             ("SA layer3 1Mx256x128 ns3 bn+relu prologue, stats epilogue", 1 << 20, 256, 128, 3, True, False),
             ("dX 16384x512x512 ns2 (MN-major W)", 16384, 512, 512, 2, False, True),
             ("dX 2048x512x512 ns2 (MN-major W)", 2048, 512, 512, 2, False, True),
             ("linear 2048x256x512 ns3 (decoder FFN1)", 2048, 256, 512, 3, False, False),
             ("SA dz1 1Mx128x256 ns2 (MN-major W)", 1 << 20, 128, 256, 2, False, True)]
    for name, m, n, k, ns, sa, mn in cases:
        if only and only not in name:
            continue
        a = torch.randn(m, k, device="cuda")
        if mn:
            w = torch.randn(k, n, device="cuda") / k ** 0.5          # forward weight (rows = contraction)
            planes = ops.pack_split(w, k, n, n, 1, 3)
        else:
            w = torch.randn(n, k, device="cuda") / k ** 0.5
            planes = ops.pack_split(w, n, k, k, 1, 3)
        out = torch.empty(m, n, device="cuda")
        if sa:
            sc, sh = torch.rand(k, device="cuda") + 0.5, torch.randn(k, device="cuda")
            fn = lambda: ops.gemm_a32(a, planes, n, mode=ops.A32_AFFINE_RELU, scale=sc, shift=sh, out=out,
                                      want_stats=True, nsplit=ns)
        else:
            fn = lambda: ops.gemm_a32(a, planes, n, out=out, b_mn=mn, nsplit=ns)
        ms = timeit(fn)
        flops = 2.0 * m * n * k
        nbytes = 4.0 * m * k + 4.0 * m * n + 2.0 * ns * n * k
        print(json.dumps({"case": name, "ms": round(ms, 4), "useful_tflops": round(flops / ms / 1e9, 1),
                          "tensor_pipe_tflops": round(flops * {2: 3, 3: 6}[ns] / ms / 1e9, 1),
                          "algorithmic_GBps": round(nbytes / ms / 1e6, 1)}))
    # weight gradient from fp32 rows
    for name, rows, m, n in [("dW 16384 rows 512x512", 16384, 512, 512), ("SA dW2 1M rows 256x128", 1 << 20, 256, 128),
                             ("SA dW1 1M rows 128x64", 1 << 20, 128, 64)]:
        if only and only not in name:
            continue
        a = torch.randn(rows, m, device="cuda")
        b = torch.randn(rows, n, device="cuda")
        ms = timeit(lambda: ops.gemm_tn32(a, b))
        print(json.dumps({"case": name, "ms": round(ms, 4), "useful_tflops": round(2.0 * rows * m * n / ms / 1e9, 1),
                          "algorithmic_GBps": round(4.0 * rows * (m + n) / ms / 1e6, 1)}))


if __name__ == "__main__":
    main()
