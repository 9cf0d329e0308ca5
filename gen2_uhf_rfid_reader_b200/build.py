"""Builds librfid_b200.so (CUDA kernels + C-ABI) in-tree with nvcc for sm_90a (H100)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "librfid_b200.so")
SOURCES = ["rfid_b200.cu"]
import glob
HEADERS = sorted(os.path.basename(h) for h in glob.glob(os.path.join(CSRC, "*.cuh"))) + ["../../include/rfid_b200.h"]

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              # no FMA contraction: the reference's x86-64 objects contain none (SURVEY.md A.5)
              "-fmad=false",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared", "-diag-suppress", "550"]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    """Compile if needed; returns the library path.  Raises if nvcc is unavailable and no library exists."""
    if not force and not _stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        if os.path.exists(LIB):
            return LIB
        raise RuntimeError("nvcc not found and %s is missing" % LIB)
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + \
          [os.path.join(CSRC, s) for s in SOURCES]
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB


def build_harness(src, lib, force=False):
    """Compile a CUDA test harness (tests/cuda/*.cu) that includes csrc headers, with the library's flags; returns lib.
    Rebuilds when stale or forced and nvcc exists; raises when there is neither nvcc nor a harness."""
    if not force and os.path.exists(lib):
        t = os.path.getmtime(lib)
        if all(os.path.getmtime(d) <= t for d in [src] + glob.glob(os.path.join(CSRC, "*.cuh"))):
            return lib
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        if os.path.exists(lib):
            return lib
        raise RuntimeError("nvcc not found and %s is missing" % lib)
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-I", CSRC, "-o", lib, src], cwd=os.path.dirname(src))
    return lib


SC16_HARNESS_SRC = os.path.join(os.path.dirname(HERE), "tests", "cuda", "sc16_harness.cu")
SC16_HARNESS = os.path.join(HERE, "libsc16_harness.so")


if __name__ == "__main__":
    print(build_library(force=True, verbose=True))
