"""TEST TOOLING ONLY: builds armada_b200/csrc/armada_round.cu with g++ against
tools/simt_emu/cuda_emu.h (a deterministic single-threaded SIMT emulator) so the kernel *logic*
can be run through the parity suite without a GPU.  Not a product path, not a fallback: nothing
under armada_b200/ loads this library."""
from __future__ import annotations

import ctypes as C
import fcntl
import os
import subprocess

from armada_b200 import abi
from armada_b200.scheduler import DeviceRound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tools", "simt_emu")
CSRC = os.path.join(ROOT, "armada_b200", "csrc")
# ARMADA_EMU_COVERAGE=1 (tools/emu_coverage.py): a --coverage build under its own name, so that the plain library
# and its build command stay as they are
COVERAGE = os.environ.get("ARMADA_EMU_COVERAGE") == "1"
EMU_LIB = os.path.join(EMU_DIR, "libarmada_b200_emu_cov.so" if COVERAGE else "libarmada_b200_emu.so")
_lib = None


def build(force: bool = False) -> None:
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".inc", ".h"))]
    srcs += [os.path.join(EMU_DIR, "cuda_emu.h"), os.path.join(ROOT, "include", "armada_b200.h")]
    def stale() -> bool:
        return not os.path.exists(EMU_LIB) or any(os.path.getmtime(p) > os.path.getmtime(EMU_LIB) for p in srcs)

    if not (force or stale()):
        return
    # pytest-xdist workers race for the build: one builds (to a temporary name, renamed into place), the others wait
    with open(EMU_LIB + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if force or stale():
            tmp = f"{EMU_LIB}.{os.getpid()}.tmp"
            # coverage: the counters are named after the output file, so it is built under its final name
            out = EMU_LIB if COVERAGE else tmp
            subprocess.run(
                ["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-DARMADA_EMU", "-x", "c++",
                 os.path.join(CSRC, "armada_round.cu"), "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-I", EMU_DIR,
                 "-o", out, "-lpthread"] + (["--coverage"] if COVERAGE else []), check=True)
            if not COVERAGE:
                os.replace(tmp, EMU_LIB)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(EMU_LIB)
        abi.declare_prototypes(_lib)
    return _lib


def emu_round() -> DeviceRound:
    return DeviceRound(0, lib=load())
