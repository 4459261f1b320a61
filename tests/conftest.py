import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
for extra in (ROOT / "tests", ROOT / "oracle"):  # oracle/: checkers only (see its headers)
    if str(extra) not in sys.path:
        sys.path.insert(0, str(extra))

os.environ.setdefault("MASTER_ADDR", "127.0.0.1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the GPU with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def built_lib():
    """The C-ABI library, built in-tree (nvcc cross-compiles without a GPU)."""
    from coda_neurips2023_b200 import build

    return build.build()
