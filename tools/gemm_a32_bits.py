"""Save C (and the column-statistics rows) of every fp32-A GEMM case of tools/gemm_a32_micro.py on seeded inputs, or
compare two such saves bit for bit.  For checking that a change of the kernel's schedule leaves the results alone:

    python tools/gemm_a32_bits.py save OUT_DIR [--root TREE]     # TREE: the source tree whose library to load
    python tools/gemm_a32_bits.py compare DIR_A DIR_B
"""
import argparse
import sys
from pathlib import Path

import torch

CASES = [("linear_16384x512x512_ns3", 16384, 512, 512, 3, False, False),
         ("linear_2048x512x512_ns3", 2048, 512, 512, 3, False, False),
         ("sa_layer2_1Mx128x64_ns3", 1 << 20, 128, 64, 3, True, False),
         ("sa_layer3_1Mx256x128_ns3", 1 << 20, 256, 128, 3, True, False),
         ("dx_16384x512x512_ns2", 16384, 512, 512, 2, False, True),
         ("dx_2048x512x512_ns2", 2048, 512, 512, 2, False, True),
         ("linear_2048x256x512_ns3", 2048, 256, 512, 3, False, False),
         ("sa_dz1_1Mx128x256_ns2", 1 << 20, 128, 256, 2, False, True)]


def save(out: Path, root: Path):
    sys.path.insert(0, str(root.resolve()))
    from coda_neurips2023_b200 import ops

    out.mkdir(parents=True, exist_ok=True)
    for i, (name, m, n, k, ns, sa, mn) in enumerate(CASES):
        g = torch.Generator(device="cuda").manual_seed(i)
        a = torch.randn(m, k, device="cuda", generator=g)
        w = torch.randn(*((k, n) if mn else (n, k)), device="cuda", generator=g) / k ** 0.5
        planes = ops.pack_split(w, *w.shape, w.shape[1], 1, 3)
        if sa:
            sc = torch.rand(k, device="cuda", generator=g) + 0.5
            sh = torch.randn(k, device="cuda", generator=g)
            c, st = ops.gemm_a32(a, planes, n, mode=ops.A32_AFFINE_RELU, scale=sc, shift=sh, want_stats=True,
                                 nsplit=ns)
            torch.save({"c": c.cpu(), "stats": st.cpu()}, out / f"{name}.pt")
        else:
            c = ops.gemm_a32(a, planes, n, b_mn=mn, nsplit=ns)
            torch.save({"c": c.cpu()}, out / f"{name}.pt")
        print("saved", name, flush=True)


def compare(da: Path, db: Path) -> int:
    bad = 0
    for name, *_ in CASES:
        x, y = torch.load(da / f"{name}.pt"), torch.load(db / f"{name}.pt")
        for key in x:
            same = torch.equal(x[key], y[key])
            bad += not same
            print(f"{name} {key}: {'bit-identical' if same else 'DIFFERENT'}")
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
