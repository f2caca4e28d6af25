"""In-tree build of libcoast_rt.so (nvcc cross-compiles sm_90a without a GPU)."""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcoast_rt.so")


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".c", ".h", ".inc", ".S"))]
    srcs.append(os.path.join(HERE, "..", "include", "coast_rt.h"))
    return any(os.path.getmtime(s) > t for s in srcs)


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile coast_kernels.cu -> sm_90a cubin and link libcoast_rt.so next to this file."""
    if force or _stale():
        cmd = ["make", "-C", CSRC] + (["-B"] if force else [])
        res = subprocess.run(cmd, capture_output=not verbose, text=True)
        if res.returncode != 0:
            raise RuntimeError("building libcoast_rt.so failed:\n" + (res.stdout or "") + (res.stderr or ""))
    return LIB
