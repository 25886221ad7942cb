"""Build libmmplace.so in-tree with nvcc for sm_90a (H100).  `python -m modelmesh_b200.build`."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(CSRC, "libmmplace.so")
SOURCES = ["mmplace.cu"]
DEPS = ["mmplace.cu", "place_core.cuh", "host_state.hpp", "scan_kernels.cuh", "commit_kernels.cuh", "churn_kernels.cuh",
        "registry_kernels.cuh", os.path.join("..", "..", "include", "mmplace.h"),
        os.path.join("..", "build.py")]  # the compiler flags below: a library built with other flags is rebuilt


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def up_to_date() -> bool:
    if not os.path.exists(SO):
        return False
    t = os.path.getmtime(SO)
    return all(os.path.getmtime(os.path.join(CSRC, d)) <= t for d in DEPS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and up_to_date():
        return SO
    cmd = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "-Xcompiler", "-fPIC", "-Xlinker", "-Bsymbolic", "-shared", "-ldl", "-o", SO] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
        print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
