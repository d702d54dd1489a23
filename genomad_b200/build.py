"""
Build libgnm.so (the sm_90a kernels + C ABI) in-tree with nvcc.

    python -m genomad_b200.build [--force]

nvcc cross-compiles for sm_90a without a GPU, so this runs on a machine without one; the resulting
genomad_b200/libgnm.so is git-ignored and rebuilt whenever a source is newer.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libgnm.so"
SOURCES = [CSRC / "api.cu", CSRC / "fasta.cpp", CSRC / "tfrecord.cpp", CSRC / "tsv.cpp"]
HEADERS = sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "gnm.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
    "-lcudart", "-Xcompiler", "-pthread", "-lz",
]


def find_nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found (needed to build libgnm.so)")


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    return any(p.stat().st_mtime > t for p in SOURCES + HEADERS + [Path(__file__)])


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    cmd = [find_nvcc(), *NVCC_FLAGS, "-o", str(LIB), *map(str, SOURCES)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    (PKG / "build.log").write_text(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed ({res.returncode}):\n{log[-4000:]}")
    if verbose:
        print(log)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
