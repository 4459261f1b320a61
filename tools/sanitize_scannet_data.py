"""Small invocation of every ScanNet data-layer kernel (coda_sample_points_ex, coda_points_flip2_rotate_scale, and the
extent / RandomCuboid / image kernels the batch reuses) at the test shapes, meant to run under compute-sanitizer
(memcheck, racecheck)."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import scannet_data_common as C  # noqa: E402
from coda_neurips2023_b200.datasets import DeviceScanNetAugmentor  # noqa: E402
from test_scannet_data_gpu import run_device  # noqa: E402

for name in C.CASES:
    aug = DeviceScanNetAugmentor(C.SELECT_RANGE, num_points=C.NUM_POINTS, random_cuboid_min_points=C.CASES[name][1],
                                 image_size=C.IMAGE_SIZE)
    run_device([C.scene(name)], C.draws(name), aug)
torch.cuda.synchronize()
print("sanitize run ok")
