"""Build libmm_b200.so (the C-ABI in include/mm_b200.h) for sm_90a with nvcc, in-tree.

    python -m models_b200.csrc.build [--force] [--verbose]

The library is written to models_b200/_lib/libmm_b200.so (git-ignored), so the package is importable from
the repository tree without an install step.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent
PKG = CSRC.parent
LIB_DIR = PKG / "_lib"
LIB = LIB_DIR / "libmm_b200.so"
OBJ_DIR = CSRC / "build"

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-O3", "--expt-relaxed-constexpr"]


def nvcc_path() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found: cannot build libmm_b200.so")
    return p


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _stale(out: Path, deps: list[Path]) -> bool:
    if not out.exists():
        return True
    t = out.stat().st_mtime
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    nvcc = nvcc_path()
    OBJ_DIR.mkdir(exist_ok=True)
    LIB_DIR.mkdir(exist_ok=True)
    headers = sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "mm_b200.h"]
    todo = []
    objs = []
    for src in sources():
        obj = OBJ_DIR / (src.stem + ".o")
        objs.append(obj)
        if force or _stale(obj, [src] + headers):
            cmd = [nvcc, *ARCH_FLAGS, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            todo.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose:
            sys.stderr.write(r.stdout + r.stderr)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(todo)))) as ex:
        list(ex.map(run, todo))
    if todo or force or _stale(LIB, objs):
        run([nvcc, *ARCH_FLAGS, "-shared", "-o", str(LIB), *map(str, objs), "-lcudart"])
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
