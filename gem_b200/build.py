"""Build the sm_90a shared library in-tree (gem_b200/lib/libgem_b200.so).

nvcc cross-compiles without a GPU.  Flags: -gencode arch=compute_90a,code=sm_90a (H100 only,
no PTX for other architectures, no multi-backend dispatch), -lineinfo (ncu source view),
-fmad=false (the arithmetic definition: no FMA contraction, see DESIGN.md).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libgem_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-fmad=false", "-std=c++17",
    "-Xcompiler", "-ffp-contract=off",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _newer(target: str, sources: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def sources() -> list[str]:
    out = []
    for d in (CSRC, os.path.join(ROOT, "include")):
        for f in sorted(os.listdir(d)):
            if f.endswith((".cu", ".cuh", ".h", ".hpp", ".cpp")):
                out.append(os.path.join(d, f))
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile libgem_b200.so (kernels + C ABI; the C++ facade is header-only)."""
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = sources()
    if force or not _newer(LIB, srcs):
        cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB, os.path.join(CSRC, "gem_api.cu")]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        subprocess.run(cmd, check=True, cwd=CSRC)
    return LIB


def build_oracle(force: bool = False) -> str:
    """Build the CPU oracle (test infrastructure; only tests/, smoke() and the bench's
    cpu_baseline legs use it)."""
    odir = os.path.join(ROOT, "oracle")
    lib = os.path.join(odir, "libgem_oracle.so")
    srcs = [os.path.join(odir, "gem_oracle.c"), os.path.join(odir, "gem_oracle.h")]
    if force or not _newer(lib, srcs):
        subprocess.run(["make", "-C", odir] + (["-B"] if force else []), check=True,
                       stdout=subprocess.DEVNULL)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
