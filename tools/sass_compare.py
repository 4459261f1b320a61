"""Compare what ptxas makes of two source trees, kernel by kernel.  For checking that a change meant to leave the
device code alone (a refactor of shared helpers) does:

    python tools/sass_compare.py PARENT_TREE BRANCH_TREE [--jobs N]

Every csrc/*.cu of both trees is compiled with build.NVCC_FLAGS plus `-cubin -Xptxas -v`.  For every kernel (name
demangled, with the anonymous namespace's per-file hash gone) it reports registers, spill stores / loads and static
shared memory as ptxas gives them, any C7515 warning (wgmma serialized), and the opcode histogram of
`cuobjdump -sass`.  Exits 1 if a kernel is missing from either tree, a resource figure differs, or a C7515 warning
appears; kernels whose opcode histograms differ are listed, with the opcodes whose counts changed.
"""
import argparse
import collections
import concurrent.futures as cf
import importlib.util
import re
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

CUDA_BIN = Path("/usr/local/cuda/bin")


def _tool(name):
    return shutil.which(name) or str(CUDA_BIN / name)


def _nvcc_flags(tree: Path):
    spec = importlib.util.spec_from_file_location("_tree_build", tree / "coda_neurips2023_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return list(mod.NVCC_FLAGS)


def _demangle(names):
    if not names:
        return {}
    out = subprocess.run([_tool("cu++filt")], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, out.stdout.splitlines()))


def _ptxas_info(log: str):
    """mangled name -> {regs, spill_st, spill_ld, smem, c7515} from `ptxas -v` output."""
    info, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
            info[cur] = {"regs": 0, "spill_st": 0, "spill_ld": 0, "smem": 0, "c7515": False}
            continue
        if "C7515" in line:
            m = re.search(r"function '([^']+)'", line)
            name = m.group(1) if m else cur
            info.setdefault(name, {"regs": 0, "spill_st": 0, "spill_ld": 0, "smem": 0, "c7515": False})["c7515"] = True
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            info[cur]["spill_st"], info[cur]["spill_ld"] = int(m.group(1)), int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            info[cur]["regs"] = int(m.group(1))
            s = re.search(r"(\d+) bytes smem", line)
            info[cur]["smem"] = int(s.group(1)) if s else 0
    return info


def _histograms(cubin: Path):
    """mangled name -> Counter of opcodes (with modifiers) of its SASS."""
    text = subprocess.run([_tool("cuobjdump"), "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    hist, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = hist.setdefault(m.group(1), collections.Counter())
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur is not None:
            toks = m.group(1).split()
            if toks and toks[0].startswith("@"):
                toks = toks[1:]
            if toks:
                cur[toks[0]] += 1
    return hist


def compile_one(src: Path, flags, work: Path):
    cubin = work / (src.stem + ".cubin")
    cmd = [_tool("nvcc"), *flags, "-cubin", "-Xptxas", "-v", str(src), "-o", str(cubin)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    info, hist = _ptxas_info(r.stdout + r.stderr), _histograms(cubin)
    names = _demangle(sorted(set(info) | set(hist)))
    kernels = {}
    for mangled in set(info) | set(hist):
        k = kernels.setdefault((src.name, names.get(mangled, mangled)), {"res": None, "hist": collections.Counter()})
        if mangled in info:
            k["res"] = info[mangled]
        if mangled in hist:
            k["hist"] = hist[mangled]
    return kernels


def collect(tree: Path, flags, jobs: int):
    srcs = sorted((tree / "coda_neurips2023_b200" / "csrc").glob("*.cu"))
    with tempfile.TemporaryDirectory() as tmp, cf.ThreadPoolExecutor(max_workers=jobs) as ex:
        work = Path(tmp)
        out = {}
        for kernels in ex.map(lambda s: compile_one(s, flags, work), srcs):
            out.update(kernels)
        return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("parent", type=Path)
    ap.add_argument("branch", type=Path)
    ap.add_argument("--jobs", type=int, default=8)
    args = ap.parse_args()
    flags = _nvcc_flags(args.branch)
    a = collect(args.parent, flags, args.jobs)
    b = collect(args.branch, flags, args.jobs)
    failed, hist_changed = False, 0
    for key in sorted(set(a) | set(b)):
        src, name = key
        label = f"{src}: {name}"
        if key not in a or key not in b:
            print(f"MISSING in {'parent' if key not in a else 'branch'}: {label}")
            failed = True
            continue
        ra, rb = a[key]["res"], b[key]["res"]
        res = rb or {}
        line = (f"{label}\n    regs {res.get('regs')}  spill st/ld {res.get('spill_st')}/{res.get('spill_ld')}  "
                f"smem {res.get('smem')}  instructions {sum(b[key]['hist'].values())}")
        status = []
        if ra != rb:
            status.append(f"RESOURCES DIFFER (parent {ra})")
            failed = True
        if (ra and ra["c7515"]) or (rb and rb["c7515"]):
            status.append("C7515 wgmma serialized")
            failed = True
        ha, hb = a[key]["hist"], b[key]["hist"]
        if ha != hb:
            hist_changed += 1
            diff = {op: hb[op] - ha[op] for op in set(ha) | set(hb) if hb[op] != ha[op]}
            status.append("HISTOGRAM DIFFERS " + " ".join(f"{op}:{d:+d}" for op, d in sorted(diff.items())))
        print(line + ("\n    " + "; ".join(status) if status else "  (same)"))
    print(f"{len(b)} kernels in branch, {len(a)} in parent; {hist_changed} opcode histograms differ; "
          f"{'FAIL' if failed else 'resources identical, no C7515'}")
    return 1 if failed else 0


if __name__ == "__main__":
    sys.exit(main())
