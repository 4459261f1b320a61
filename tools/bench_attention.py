"""Micro-benchmark of the fused attention kernels on the training step's shapes (H100).

    python tools/bench_attention.py            # forward: one JSON line per case
    python tools/bench_attention.py --bwd      # backward (coda_attention_bwd_ex): one JSON line per case

Backward lines give the whole call (operand packing + D + both kernels) timed with CUDA events, and the dQ and
dK/dV kernels on their own from a separate torch.profiler run.  Work per backward (bh = b*h, n = lq*lk*hd):
algorithmic 10*bh*n (the five products S, dP, dV, dK, dQ), tensor pipe 42*bh*n (S and dP are recomputed in both
kernels: 7 products, each 3 bf16 plane products); the dQ kernel does 18*bh*n of it, the dK/dV kernel 24*bh*n.
"""
import argparse
import ctypes
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from coda_neurips2023_b200 import _lib  # noqa: E402

CASES = [  # name, b, h, lq, lk, hd, nsplit, dropout
    ("encoder self (drop 0.1)", 8, 4, 2048, 2048, 64, 3, 0.1),
    ("encoder self (no drop)", 8, 4, 2048, 2048, 64, 3, 0.0),
    ("encoder self 2 planes", 8, 4, 2048, 2048, 64, 2, 0.1),
    ("decoder cross", 8, 4, 256, 2048, 128, 3, 0.1),
    ("decoder self", 8, 4, 256, 256, 128, 3, 0.1),
    ("clip image tower", 256, 12, 50, 50, 64, 2, 0.0),
]

BWD_CASES = [  # name, b, h, lq, lk, hd, dropout, launches per training step
    ("encoder self", 8, 4, 2048, 2048, 64, 0.1, 3),
    ("decoder cross", 8, 4, 256, 2048, 128, 0.1, 8),
    ("decoder self", 8, 4, 256, 256, 128, 0.1, 8),
]

P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731


def event_ms(fn, reps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def bench_fwd(L, dev, stream, cases):
    for name, b, h, lq, lk, hd, ns, drop in cases:
        q = torch.randn(lq, b, h * hd, device=dev)
        k = torch.randn(lk, b, h * hd, device=dev)
        v = torch.randn(lk, b, h * hd, device=dev)
        ws = torch.empty(int(L.coda_attention_workspace_bytes(b, h, lq, lk, hd, ns)), dtype=torch.uint8, device=dev)
        out = torch.empty_like(q)
        lse = torch.empty(b * h, lq, device=dev)
        _lib.check(L.coda_attention_pack(b, h, lq, lk, hd, ns, ctypes.c_float(hd ** -0.5), P(q), P(k), P(v), P(ws),
                                         stream), "pack")

        def launch():
            return L.coda_attention_fwd_packed(b, h, lq, lk, hd, ns, P(ws), P(out), P(lse), ctypes.c_float(drop), 7,
                                               None, stream)

        for _ in range(3):
            _lib.check(launch(), "fwd")
        ms = event_ms(launch, 20)
        flops = 4.0 * b * h * lq * lk * hd
        print(json.dumps({"case": name, "b": b, "h": h, "lq": lq, "lk": lk, "hd": hd, "nsplit": ns, "dropout": drop,
                          "ms": round(ms, 4), "algorithmic_tflops": round(flops / ms / 1e9, 1)}))


def bench_bwd(L, dev, stream, cases, reps):
    from torch.profiler import ProfilerActivity, profile

    L.coda_attention_bwd_workspace_bytes.restype = ctypes.c_longlong
    for name, b, h, lq, lk, hd, drop, per_step in cases:
        e = h * hd
        q = torch.randn(lq, b, e, device=dev)
        k = torch.randn(lk, b, e, device=dev)
        v = torch.randn(lk, b, e, device=dev)
        dout = torch.randn(lq, b, e, device=dev)
        out = torch.empty_like(q)
        lse = torch.empty(b * h, lq, device=dev)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        scale = ctypes.c_float(hd ** -0.5)
        # the forward with the same dropout stream gives the out / lse the backward is run on in the step
        fws = torch.empty(int(L.coda_attention_workspace_bytes(b, h, lq, lk, hd, 3)), dtype=torch.uint8, device=dev)
        _lib.check(L.coda_attention_pack(b, h, lq, lk, hd, 3, scale, P(q), P(k), P(v), P(fws), stream), "pack")
        _lib.check(L.coda_attention_fwd_packed(b, h, lq, lk, hd, 3, P(fws), P(out), P(lse), ctypes.c_float(drop), 7,
                                               None, stream), "fwd")
        bws = torch.empty(int(L.coda_attention_bwd_workspace_bytes(b, h, lq, lk, hd)), dtype=torch.uint8, device=dev)
        cl = ctypes.c_longlong

        def launch():
            return L.coda_attention_bwd_ex(b, h, lq, lk, hd, scale, P(q), P(k), P(v), cl(e), cl(e), cl(e), P(out),
                                           P(dout), P(lse), P(dq), P(dk), P(dv), cl(e), cl(e), cl(e), None, None,
                                           ctypes.c_float(drop), 7, None, P(bws), stream)

        for _ in range(3):
            _lib.check(launch(), "bwd")
        ms = event_ms(launch, reps)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                launch()
            torch.cuda.synchronize()
        kern = {"dq": 0.0, "dkv": 0.0}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            if "attn_bwd_dq_kernel" in ev.key:
                kern["dq"] += t / 1e3 / reps
            elif "attn_bwd_dkv_kernel" in ev.key:
                kern["dkv"] += t / 1e3 / reps
        n = float(b * h) * lq * lk * hd
        tf = lambda flop, t: round(flop / t / 1e9, 1) if t > 0 else None  # noqa: E731
        print(json.dumps({
            "case": name, "b": b, "h": h, "lq": lq, "lk": lk, "hd": hd, "dropout": drop, "per_step": per_step,
            "ms_call": round(ms, 4), "algorithmic_tflops": tf(10 * n, ms), "pipe_tflops": tf(42 * n, ms),
            "ms_dq": round(kern["dq"], 4), "dq_pipe_tflops": tf(18 * n, kern["dq"]),
            "ms_dkv": round(kern["dkv"], 4), "dkv_pipe_tflops": tf(24 * n, kern["dkv"]),
            "ms_kernels": round(kern["dq"] + kern["dkv"], 4), "kernels_pipe_tflops": tf(42 * n, kern["dq"] + kern["dkv"]),
            "ms_per_step": round(ms * per_step, 3)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("cases", nargs="*", type=int, help="case indices (default: all)")
    ap.add_argument("--bwd", action="store_true", help="time the backward instead of the forward")
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    L = _lib.lib()
    L.coda_attention_workspace_bytes.restype = ctypes.c_longlong
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    table = BWD_CASES if a.bwd else CASES
    cases = [table[i] for i in a.cases] if a.cases else table
    if a.bwd:
        bench_bwd(L, dev, stream, cases, a.reps)
    else:
        bench_fwd(L, dev, stream, cases)


if __name__ == "__main__":
    main()
