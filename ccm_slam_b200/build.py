"""Builds libccm_b200.so (sm_90a, H100) in-tree with nvcc.  Used by __graft_entry__.build() and by developers.

The shared object is git-ignored; nvcc cross-compiles it without a GPU.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libccm_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--use_fast_math=false",
         "-Xcompiler", "-ffp-contract=off",
         "-Xcompiler", "-fPIC,-O3,-Wall", "-shared", "-lcudart", "-ldl"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(HERE, "..", "include", "*.h")) + [__file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    flags = [f for f in FLAGS if f != "--use_fast_math=false"]
    cmd = [NVCC] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + sources()
    print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
