"""Host emulations of the native operators: ``<name>_emulation.cpp`` includes the operator's .cu and compiles it with g++
behind the fake CUDA runtime in ``cuda_shim/``, so the library's own host code drives its kernels, one lane at a time, on
machines without a GPU."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
# -ffp-contract=off: a * b + c is not fused, as the __fmul_rn / __dmul_rn family guarantees on the device
FLAGS = ["-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wno-unknown-pragmas",
         "-I", os.path.join(HERE, "cuda_shim"), "-I", os.path.join(ROOT, "include")]


def build(name: str, tmp_path_factory) -> C.CDLL:
    """Compiles ``<name>_emulation.cpp`` into a shared library (skips the test when g++ is missing)."""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    out = tmp_path_factory.mktemp(f"{name}_emu") / f"lib{name}_emu.so"
    subprocess.run([gxx, *FLAGS, os.path.join(HERE, f"{name}_emulation.cpp"), "-o", str(out)], check=True)
    lib = C.CDLL(str(out))
    lib.cfb_last_error.restype = C.c_char_p
    return lib
