"""In-tree build of the CUDA library (sm_90a, H100) with plain nvcc.

The product is ONE C-ABI shared library, ``csrc/libcoda_b200.so``; it has no
torch / pybind dependency, so a full rebuild takes seconds and the same binary
travels to the GPU box with the repo snapshot.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
LIB = CSRC / "libcoda_b200.so"
OBJ_DIR = CSRC / "build"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; the coda_b200 CUDA library cannot be built")
    return nvcc


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def sources():
    return sorted(CSRC.glob("*.cu"))


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every ``csrc/*.cu`` for sm_90a and link ``libcoda_b200.so``."""
    srcs = sources()
    hdrs = sorted(CSRC.glob("*.cuh")) + sorted((CSRC.parent.parent / "include").glob("*.h"))
    stamp = OBJ_DIR / "stamp.txt"
    digest = _digest(srcs + hdrs)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB
    OBJ_DIR.mkdir(exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: Path) -> Path:
        obj = OBJ_DIR / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
