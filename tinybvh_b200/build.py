"""Compile the sm_90a engine in-tree: tinybvh_b200/csrc/*.cu -> tinybvh_b200/libtinybvh_b200.so (C-ABI of
include/tinybvh_b200.h).  nvcc cross-compiles without a GPU; the .so travels to the GPU box with the snapshot."""
from __future__ import annotations

import glob
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
SO = os.path.join(HERE, "libtinybvh_b200.so")
DEVICE_HEADER = os.path.join(REPO, "include", "tinybvh_b200_device.cuh")  # the walks, shared with callers' kernels
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared", "--use_fast_math=false"]
NVCC_FLAGS = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]  # never fast-math: parity is bit-exact


def sources():
    return sorted(glob.glob(os.path.join(HERE, "csrc", "*.cu")))


def stale() -> bool:
    if not os.path.isfile(SO):
        return True
    t = os.path.getmtime(SO)
    deps = (sources() + glob.glob(os.path.join(HERE, "csrc", "*.cuh")) + [os.path.join(REPO, "include", "tinybvh_b200.h"), DEVICE_HEADER]
            + glob.glob(os.path.join(REPO, "include", "tinybvh_b200_device", "*.cuh")))
    return any(os.path.getmtime(d) > t for d in deps)


def nvcc_path():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return p if os.path.isfile(p) else None


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return SO
    nvcc = nvcc_path()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libtinybvh_b200.so (there is no CPU fallback)")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + sources() + ["-o", SO + ".tmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose:
        print(r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    os.replace(SO + ".tmp", SO)
    return SO


GEN_SO = os.path.join(HERE, "libtbvh_raygen.so")


def build_raygen(force: bool = False) -> str:
    """The host-side workload generator (hostgen/raygen.c): plain C + OpenMP, float32 with contraction off so the rays are the
    ones tinybvh_b200/rays.py computes."""
    src = os.path.join(HERE, "hostgen", "raygen.c")
    if not force and os.path.isfile(GEN_SO) and os.path.getmtime(GEN_SO) >= os.path.getmtime(src):
        return GEN_SO
    cmd = ["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", src, "-lm", "-o", GEN_SO + ".tmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gcc failed:\n" + r.stdout + r.stderr)
    os.replace(GEN_SO + ".tmp", GEN_SO)
    return GEN_SO


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_raygen(force="--force" in sys.argv))
