"""Generates tests/golden/pointnet2_ref_*.npz from the REFERENCE's own CUDA extension.

Run on a GPU (the reference extension has no CPU path), with the extension built by oracle/build_ref_ext.py:
    python tests/golden/make_pointnet2_golden.py [OUT_DIR]        (default: tests/golden/)  Inputs are regenerated from the seed by
coda_neurips2023_b200.synthetic.point_clouds, so only outputs are stored.
"""
import importlib
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "_ref"))
from coda_neurips2023_b200 import synthetic  # noqa: E402

ref = importlib.import_module("pointnet2._ext")

CASES = [
    # name, batch, n, m, seed, dup_frac, radius, nsample, nn_unknown, nn_known
    ("small", 2, 3000, 256, 101, 0.2, 0.3, 16, 500, 200),
    ("tiny_ties", 3, 300, 64, 102, 0.5, 0.5, 8, 100, 2),
    ("sunrgbd", 1, 20000, 2048, 103, 0.01, 0.2, 64, 1000, 512),
    ("queries", 2, 2048, 256, 104, 0.05, 0.2, 32, 2048, 256),
]


def main(out_dir: str):
    out = Path(out_dir)
    out.mkdir(parents=True, exist_ok=True)
    for name, b, n, m, seed, dup, radius, ns, nu, nk in CASES:
        xyz = torch.from_numpy(synthetic.point_clouds(b, n, seed=seed, dup_frac=dup)).cuda()
        fps = ref.furthest_point_sampling(xyz, m)
        new_xyz = torch.gather(xyz, 1, fps.long()[..., None].expand(-1, -1, 3)).contiguous()
        ball = ref.ball_query(new_xyz, xyz, radius, ns)
        d2, nn = ref.three_nn(xyz[:, :nu].contiguous(), new_xyz[:, :nk].contiguous())
        np.savez_compressed(
            out / f"pointnet2_ref_{name}.npz", batch=b, n=n, m=m, seed=seed, dup_frac=dup, radius=radius,
            nsample=ns, nn_unknown=nu, nn_known=nk, fps_idx=fps.cpu().numpy(), ball_idx=ball.cpu().numpy(),
            nn_idx=nn.cpu().numpy(), nn_dist2=d2.cpu().numpy())
        print("wrote", name)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else str(Path(__file__).resolve().parent))
