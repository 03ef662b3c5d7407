"""Build libmmfs_b200.so in-tree with nvcc for sm_90a (no torch headers involved).

    python mm-interleaved_b200/build.py [--force]

The library lands next to this file, so the package imports from the repository tree;
it is git-ignored (built artefact).
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmmfs_b200.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + \
        glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    flags = list(NVCC_FLAGS)
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [nvcc, *flags, "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd)))
    for src, p in procs:
        if p.wait() != 0:
            raise RuntimeError(f"nvcc failed on {src}")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB, *objs, "-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
