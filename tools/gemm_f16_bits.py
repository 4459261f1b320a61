"""Save C of every CLIP tower fp16 GEMM of tools/bench_gemm_fp16.py (with its epilogue) on seeded inputs, or compare
two such saves bit for bit.  For checking that a change of the kernel's schedule leaves the results alone:

    python tools/gemm_f16_bits.py save OUT_DIR [--root TREE]     # TREE: the source tree whose library to load
    python tools/gemm_f16_bits.py compare DIR_A DIR_B
"""
import argparse
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_gemm_fp16 import SHAPES  # noqa: E402


def save(out: Path, root: Path):
    sys.path.insert(0, str(root.resolve()))
    from coda_neurips2023_b200 import ops

    out.mkdir(parents=True, exist_ok=True)
    for i, (name, m, n, k, bias, act, res) in enumerate(SHAPES):
        g = torch.Generator(device="cuda").manual_seed(i)
        a = (torch.randn(1, 1, m, k, device="cuda", generator=g) * 0.5).half()
        b = (torch.randn(1, 1, n, k, device="cuda", generator=g) * k ** -0.5).half()
        bv = torch.randn(n, device="cuda", generator=g) if bias else None
        r = torch.randn(m, n, device="cuda", generator=g).half() if res else None
        c = ops.gemm_nt(a, b, m, n, bias=bv, act=act, out_dtype=torch.float16, residual=r)
        torch.save({"c": c.cpu()}, out / f"{name}.pt")
        print("saved", name, flush=True)


def compare(da: Path, db: Path) -> int:
    bad = 0
    for name, *_ in SHAPES:
        x, y = torch.load(da / f"{name}.pt")["c"], torch.load(db / f"{name}.pt")["c"]
        same = torch.equal(x, y)
        bad += not same
        msg = "bit-identical"
        if not same:
            # largest difference in units of the last place of the fp16 values
            ix, iy = x.view(torch.int16).int(), y.view(torch.int16).int()
            msg = f"DIFFERENT: {int((x != y).sum())} elements, max {int((ix - iy).abs().max())} ulp"
        print(f"{name} c: {msg}")
    return bad


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("cmd", choices=["save", "compare"])
    ap.add_argument("dirs", nargs="+", type=Path)
    ap.add_argument("--root", type=Path, default=Path(__file__).resolve().parents[1])
    args = ap.parse_args()
    if args.cmd == "save":
        save(args.dirs[0], args.root)
    else:
        sys.exit(1 if compare(*args.dirs) else 0)
