"""Build libwmd.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m wavelet_monodepth_b200.build [--force] [--verbose]

The shared library is a build product (git-ignored); build() or this module rebuilds it whenever a source is newer.
"""
import glob
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libwmd.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "shared",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _deps():
    return sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(REPO, "include", "*.h"))


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in _deps())


def nvcc_path():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def build(force=False, verbose=False):
    """Compile every CUDA source into wavelet_monodepth_b200/libwmd.so; returns the path."""
    if not force and not is_stale():
        return LIB
    nvcc = nvcc_path()
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libwmd.so")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
          ["-I", os.path.join(REPO, "include"), "-I", CSRC, "-o", LIB] + sources()
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed (exit %d)" % res.returncode)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
