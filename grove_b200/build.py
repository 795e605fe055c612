"""In-tree build of libgrove_place.so (nvcc, sm_90a only)."""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgrove_place.so")
SOURCES = ["engine.cu"]
DEPS = ["engine.cu", "kernels.cuh", "common.cuh", "tables.cuh", "fit.cuh", "score.cuh", "admit.cuh", "relax.cuh",
        "reclaim.cuh", "donor.cuh", "fairshare.cuh", "overquota.cuh", "diagnose.cuh", "spread.cuh", "fence.cuh", "consolidate.cuh", "queue.cuh", "binpack.cuh", "imex.cuh", os.path.join("..", "..", "include", "grove_place.h")]
NVCC_FLAGS = [
    "-DGROVE_INLINE_ALL",
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-Xcompiler", "-fopenmp", "-shared", "-cudart", "shared", "-lgomp",
]


def nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    # this file holds the flags: a library built with other flags (another architecture) is stale too
    return os.path.getmtime(__file__) > t or any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


def build(force: bool = False, verbose: bool = False) -> str:
    if force or stale():
        cmd = [nvcc(), *NVCC_FLAGS, "-o", LIB, *[os.path.join(CSRC, s) for s in SOURCES]]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        env = dict(os.environ)
        env.pop("CC", None); env.pop("CXX", None)  # a CC/CXX wrapper without libgomp specs would break -fopenmp
        subprocess.check_call(cmd, env=env)
    return LIB


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
