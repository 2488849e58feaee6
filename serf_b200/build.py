"""Builds serf_b200/libserfsim.so (CUDA kernels + C ABI) in-tree for sm_90a with nvcc."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libserfsim.so")
SOURCES = ["serfsim.cu", "tick_kernel.cu", "uevent_kernel.cu", "byz_kernel.cu", "wire_codec.cu"]
HEADERS = ["record.cuh", "uevent.cuh", "byz.cuh", "tick_kernel.cuh", "wire.cuh", os.path.join("..", "..", "include", "serfsim.h")]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built")


def is_stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not is_stale():
        return OUT
    cmd = [nvcc_path(), "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
           "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-shared", "-o", OUT]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += [os.path.join(CSRC, s) for s in SOURCES]
    subprocess.check_call(cmd, cwd=CSRC)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
