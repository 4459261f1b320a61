"""Micro-benchmark of the fused attention kernels on the training step's shapes (H100).

    python tools/bench_attention.py            # one JSON line per case
"""
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


def main():
    dev = torch.device("cuda:0")
    L = _lib.lib()
    L.coda_attention_workspace_bytes.restype = ctypes.c_longlong
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    cases = CASES if len(sys.argv) < 2 else [CASES[int(i)] for i in sys.argv[1:]]   # e.g. `0` under ncu
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
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 20
        e0.record()
        for _ in range(reps):
            launch()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        flops = 4.0 * b * h * lq * lk * hd
        print(json.dumps({"case": name, "b": b, "h": h, "lq": lq, "lk": lk, "hd": hd, "nsplit": ns, "dropout": drop,
                          "ms": round(ms, 4), "algorithmic_tflops": round(flops / ms / 1e9, 1)}))


if __name__ == "__main__":
    main()
