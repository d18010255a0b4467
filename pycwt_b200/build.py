"""Builds the CUDA engine (sm_90a, H100) in-tree: pycwt_b200/libcwtb200.so.

nvcc cross-compiles without a GPU.  The library is a plain C-ABI shared object
(include/cwt_b200.h); no PyTorch involved.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "csrc", "engine.cu")
DEPS = [os.path.join(HERE, "csrc", f) for f in
        ("engine.cu", "kernels.cuh", "fft_tile.cuh", "cplx.cuh")] + \
       [os.path.join(ROOT, "include", "cwt_b200.h")]
LIB = os.path.join(HERE, "libcwtb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-std=c++17", "-O3", "-lineinfo",
         "-gencode", "arch=compute_90a,code=sm_90a",
         "-Xcompiler", "-fPIC", "-shared"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile the engine if sources are newer than the library. Returns its path."""
    if force or _stale(LIB, DEPS):
        cmd = [NVCC] + FLAGS + [SRC, "-o", LIB]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return LIB


def build_emulation(out_dir, force=False):
    """TESTS ONLY: the same sources compiled with -DCWTB_HOST_EMU, so the kernel bodies
    run as plain C++ loops on the CPU.  Never loaded by the package."""
    os.makedirs(out_dir, exist_ok=True)
    lib = os.path.join(out_dir, "libcwtb200_emu.so")
    if force or _stale(lib, DEPS):
        subprocess.check_call([NVCC, "-std=c++17", "-O2", "-DCWTB_HOST_EMU", "-w",
                               "-Xcompiler", "-fPIC", "-shared", SRC, "-o", lib])
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
