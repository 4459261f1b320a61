"""Compile the REFERENCE's own pointnet2 CUDA extension, unmodified, for use as a checker.

TEST INFRASTRUCTURE ONLY (see oracle/pointnet2_oracle.c header).

Sources are compiled where they lie under
/root/reference/third_party_pointnet2/pointnet2/_ext_src (never copied); the
only outputs are ``oracle/_ref/pointnet2/_ext.so`` and an empty
``oracle/_ref/pointnet2/__init__.py`` (``oracle/_ref/`` is git-ignored; where the
reference sources are absent, a prebuilt ``oracle/_ref`` is kept, and the GPU tests
load it as ``pointnet2._ext`` to compare our kernels against it).

This is a short recipe of direct nvcc / g++ calls -- the reference's own
setup.py is not run.  The reference passes only ``-O2`` (setup.py:26-29) and gets
its arch from torch; we pin ``compute_90/sm_90`` (plain, not 'a': the
reference has no arch-specific code).
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys
from pathlib import Path

REF_SRC = Path("/root/reference/third_party_pointnet2/pointnet2/_ext_src")
OUT = Path(__file__).resolve().parent / "_ref" / "pointnet2"
OBJ = OUT.parent / "obj"


def main() -> int:
    if not os.path.isdir(REF_SRC):
        print("reference sources not present; keeping any prebuilt oracle/_ref", file=sys.stderr)
        return 0
    so = OUT / "_ext.so"
    srcs = sorted((REF_SRC / "src").glob("*.cpp")) + sorted((REF_SRC / "src").glob("*.cu"))
    if so.exists() and all(so.stat().st_mtime > s.stat().st_mtime for s in srcs):
        print(so)
        return 0
    from torch.utils import cpp_extension as ce
    import sysconfig

    OUT.mkdir(parents=True, exist_ok=True)
    OBJ.mkdir(parents=True, exist_ok=True)
    inc = [f"-I{REF_SRC / 'include'}"] + [f"-I{p}" for p in ce.include_paths("cuda")]
    inc.append(f"-I{sysconfig.get_paths()['include']}")
    common = ["-O2", "-std=c++17", "-DTORCH_EXTENSION_NAME=_ext", "-DTORCH_API_INCLUDE_EXTENSION_H",
              "-D_GLIBCXX_USE_CXX11_ABI=1"]

    def cc(src: Path) -> Path:
        obj = OBJ / (src.name + ".o")
        if src.suffix == ".cu":
            cmd = ["nvcc", "-gencode", "arch=compute_90,code=sm_90", "-Xcompiler", "-fPIC",
                   "--expt-relaxed-constexpr", *common, *inc, "-c", str(src), "-o", str(obj)]
        else:
            cmd = ["g++", "-fPIC", *common, *inc, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
        return obj

    with cf.ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(cc, srcs))
    libs = [f"-L{p}" for p in ce.library_paths("cuda")]
    rpath = [f"-Wl,-rpath,{p}" for p in ce.library_paths("cuda")]
    cmd = ["g++", "-shared", "-o", str(so), *map(str, objs), *libs, *rpath,
           "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    (OUT / "__init__.py").write_text("")
    print(so)
    return 0


if __name__ == "__main__":
    sys.exit(main())
