"""TEST INFRASTRUCTURE -- builds and loads tests/cuda/gate_harness.cu: the gate functions of csrc/rx_gate.cuh, compiled
unchanged with the library's nvcc flags, one warp per case (tests/test_gate_fsm.py).

Only tests/ and __graft_entry__.build() may import this.
"""
import ctypes as C
import glob
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(ROOT, "tests", "cuda", "gate_harness.cu")
CSRC = os.path.join(ROOT, "gen2_uhf_rfid_reader_b200", "csrc")
LIB = os.path.join(HERE, "libgate_harness.so")


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return nvcc if os.path.exists(nvcc) else None


def command(lib=LIB, csrc=CSRC):
    """the nvcc command line: the library's flags (build.NVCC_FLAGS, -fmad=false included); the headers from csrc first,
    then from the library's csrc (so csrc may hold a modified rx_gate.cuh alone)"""
    from gen2_uhf_rfid_reader_b200.build import NVCC_FLAGS
    return [_nvcc() or "nvcc"] + NVCC_FLAGS + ["-I", csrc, "-I", CSRC, "-o", lib, SRC]


def stale(lib=LIB, csrc=CSRC):
    """True when lib is missing or older than the harness source or any header it may include"""
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    deps = [SRC] + glob.glob(os.path.join(csrc, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.cuh"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, lib=LIB, csrc=CSRC):
    """compile when stale (or forced) and nvcc exists; returns lib.  Raises when there is neither nvcc nor a harness."""
    if not force and not stale(lib, csrc):
        return lib
    if _nvcc() is None:
        if os.path.exists(lib):
            return lib
        raise RuntimeError("nvcc not found and %s is missing" % lib)
    subprocess.check_call(command(lib, csrc), cwd=os.path.dirname(SRC))
    return lib


def load(lib=LIB):
    """the harness library, rebuilt first when it is stale and nvcc exists; a missing harness is an error"""
    build(lib=lib)
    h = C.CDLL(lib)
    P, I = C.c_void_p, C.c_int
    h.gate_harness_masks.argtypes = [I, P, P, P, P, P, I]
    h.gate_harness_closed_run.argtypes = [I, P, P, P, P, I]
    h.gate_harness_stream.argtypes = [I, P, P, P, P, I, P, I, P, I]
    for f in (h.gate_harness_masks, h.gate_harness_closed_run, h.gate_harness_stream):
        f.restype = I
    return h
