"""Writes tests/golden/random_cuboid_ref.npz: the points and boxes the reference's RandomCuboid
(utils/random_cuboid.py, imported unmodified through _reference_harness) keeps when its np.random.rand /
np.random.choice draws are replaced by the replay table tests/test_data_cpu.py feeds the restatement.

    python tests/golden/make_random_cuboid_golden.py        (needs the reference checkout)
"""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent.parent / "oracle"))
import _reference_harness as H  # noqa: E402
import data_ref  # noqa: E402
from test_data_cpu import CASES, replay_table, scene  # noqa: E402


def main():
    rc = H.load("utils.random_cuboid")
    out = {}
    for seed, min_points in CASES:
        pts, boxes = scene(seed)
        crop_range, center_u = replay_table(seed)

        class Replay:
            k = -1

            @classmethod
            def rand(cls, n):
                cls.k += 1
                return (crop_range[cls.k] - 0.5) * 2.0       # exact: min_crop + r * (max_crop - min_crop) = crop_range

            @classmethod
            def choice(cls, n):
                return data_ref.center_index(center_u[cls.k], n)

        aug = rc.RandomCuboid(min_points=min_points, aspect=0.8, min_crop=0.5, max_crop=1.0)
        saved = rc.np.random.rand, rc.np.random.choice
        rc.np.random.rand, rc.np.random.choice = Replay.rand, Replay.choice
        try:
            ref_pts, ref_boxes, _ = aug(pts.copy(), boxes.copy())
        finally:
            rc.np.random.rand, rc.np.random.choice = saved
        out[f"pts_{seed}_{min_points}"] = np.asarray(ref_pts, np.float32)
        out[f"boxes_{seed}_{min_points}"] = np.asarray(ref_boxes, np.float32)
    np.savez_compressed(HERE / "random_cuboid_ref.npz", **out)


if __name__ == "__main__":
    main()
