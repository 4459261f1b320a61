"""Throughput of the wgmma GEMM (packed operands resident) vs torch.matmul fp32 / bf16."""
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from coda_neurips2023_b200 import ops  # noqa: E402


def timeit(fn, reps=20, warm=3, graph=True):
    """Per-call device time.  With graph=True the calls are replayed from a CUDA graph, so the
    host cost of a launch (ctypes, tensor-map encoding) is not part of the number -- as in the training step."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    if graph:
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            with torch.cuda.graph(g, stream=side):
                for _ in range(reps):
                    fn()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


for (m, n, k) in [(16384, 768, 256), (16384, 512, 512), (16384, 1024, 512), (8192, 8192, 8192), (1048576, 128, 64),
                  (1048576, 256, 128), (12800, 3072, 768)]:
    a = torch.randn(m, k, device="cuda")
    b = torch.randn(n, k, device="cuda")
    row = {"m": m, "n": n, "k": k}
    for ns in (1, 2, 3):
        ap, bp = ops.pack_split(a, m, k, k, 1, ns), ops.pack_split(b, n, k, k, 1, ns)
        out = torch.empty(1, m, n, device="cuda")
        ms = timeit(lambda: ops.gemm_nt(ap, bp, m, n, out=out))
        row[f"split{ns}_ms"] = round(ms, 4)
        row[f"split{ns}_tflops_useful"] = round(2.0 * m * n * k / ms / 1e9, 1)
    row["pack_a_ms"] = round(timeit(lambda: ops.pack_split(a, m, k, k, 1, 2)), 4)
    row["torch_fp32_ms"] = round(timeit(lambda: a @ b.t()), 4)
    ah, bh = a.bfloat16(), b.bfloat16()
    row["torch_bf16_ms"] = round(timeit(lambda: ah @ bh.t()), 4)
    x = a.requires_grad_(True)
    w = b.requires_grad_(True)
    def fb():
        y = ops.linear(x, w)
        y.backward(y)
    row["linear_fwd_bwd_ms"] = round(timeit(fb, reps=5, graph=False), 4)
    def fb_t():
        y = torch.nn.functional.linear(x, w)
        y.backward(y)
    row["torch_linear_fwd_bwd_ms"] = round(timeit(fb_t, reps=5, graph=False), 4)
    print(json.dumps(row), flush=True)
