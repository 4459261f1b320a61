"""Writes tests/golden/model_eval_small_gpu_bits.npz: the CoDA head's eval-mode outputs on the GPU (the `eval_small`
case of tests/model_eval_common.py: weights and running statistics filled by name, one seeded batch,
forward(if_real_test=True)), stored bit for bit.  It was run on an NVIDIA H100 80GB HBM3 from the tree of the commit
before the 3DETR + CLIP baseline head was built on the CoDA head's class, so that tests/test_baseline_eval_gpu.py can
check that the CoDA head computes the same bits as it did before.

    python tests/golden/make_coda_eval_bits_golden.py OUT.npz        (from the root of the tree to pin; needs a GPU)
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path.cwd()
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import model_eval_common as mec  # noqa: E402


def main():
    out, _ = mec.run("eval_small", "cuda")
    np.savez_compressed(sys.argv[1], **mec.blob(out))
    print("wrote", sys.argv[1], flush=True)


if __name__ == "__main__":
    main()
