"""Builds the CUDA library in-tree with nvcc for sm_90a (no JIT cache, so the .so travels with the repo)."""
from __future__ import annotations

import os
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "lib" / "libadcensus_b200.so"


def _stale() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    srcs = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list(CSRC.glob("*.cpp")) + \
        list((PKG.parent / "include").glob("*.h")) + [CSRC / "Makefile"]
    return any(s.stat().st_mtime > t for s in srcs)


def build_library(force: bool = False, verbose: bool = False) -> Path:
    """nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo ... (see csrc/Makefile)."""
    if force or _stale():
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        if not Path(nvcc).exists():
            raise RuntimeError(f"nvcc not found at {nvcc}: cannot build {LIB}")
        args = ["make", "-C", str(CSRC), f"NVCC={nvcc}", "-j8"]
        if force:
            args.insert(1, "-B")
        r = subprocess.run(args, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            print(r.stdout[-4000:])
            print(r.stderr[-4000:])
        if r.returncode != 0:
            raise RuntimeError("building libadcensus_b200.so failed")
    return LIB
