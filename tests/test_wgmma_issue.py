"""The wgmma convolutions keep their products in flight: a compile-time check, no GPU needed.

ptxas falls back to issuing every wgmma.mma_async of a kernel one at a time (a full `WARPGROUP.DEPBAR.LE gsb0, 0x0`
after each GMMA) when it cannot prove the asynchronous pipeline safe, and says so only as an info message.  Causes met
so far: a wgmma behind a runtime tile guard (C7520), a function call such as printf anywhere in the kernel (C7510), and
accumulators zeroed by register moves instead of the first product's scale-d = 0 (C7518).  This test compiles
kernels_wgmma.cu for sm_90a and reads both the ptxas messages and the SASS.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "chunkflow_b200", "csrc")


def _tool(name):
    return shutil.which(name) or next((p for p in (f"/usr/local/cuda/bin/{name}",) if os.path.exists(p)), None)


NVCC, CUOBJDUMP = _tool("nvcc"), _tool("cuobjdump")
pytestmark = pytest.mark.skipif(NVCC is None or CUOBJDUMP is None, reason="needs nvcc and cuobjdump")

F16F8, CONV, POOL, CONVT = 3, 0, 1, 2
# default-mode (f16f8) kernels whose taps must issue back to back: (cin, cout, tail, mode)
PIPELINED = {
    "16->16": (16, 16, 0, CONV),
    "16->16 pool": (16, 16, 0, POOL),
    "16->16 head+blend tail": (16, 16, 1, CONV),
    "32->16": (32, 16, 0, CONV),
    "64->32 transposed": (64, 32, 0, CONVT),
    "32->16 transposed": (32, 16, 0, CONVT),
}
# still serialized by ptxas (C7518) when Cout >= 32; strict, so that a fix has to move them up
NOT_YET = {
    "16->32": (16, 32, 0, CONV),
    "32->32": (32, 32, 0, CONV),
    "32->32 pool": (32, 32, 0, POOL),
    "32->64": (32, 64, 0, CONV),
    "64->64": (64, 64, 0, CONV),
    "64->32": (64, 32, 0, CONV),
}


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    out = tmp_path_factory.mktemp("wgmma")
    cubin = str(out / "kernels_wgmma.cubin")
    res = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
                          "-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-cubin",
                          os.path.join(CSRC, "kernels_wgmma.cu"), "-o", cubin], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    sass = subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for block in re.split(r"\n\s*Function : ", sass)[1:]:
        m = re.search(r"conv3_wgmma_kernelILi(\d+)ELi(\d+)ELi(\d)ELb(\d)ELi(\d)E", block.split("\n", 1)[0])
        if m:
            kernels[tuple(int(g) for g in m.groups())] = [l for l in block.split("\n") if "/*" in l and "*/" in l]
    return res.stdout + res.stderr, kernels


def serialized_products(lines):
    """(GMMA count, how many GMMAs wait for all earlier products: a full DEPBAR since the previous GMMA, no barrier between)"""
    n = waits = 0
    full_wait = False
    for line in lines:
        if "gdesc[URZ]" in line:  # the empty placeholder ptxas emits for a commit group with no products
            continue
        if re.search(r"\b[HQIB]GMMA\.", line):
            n += 1
            waits += full_wait
            full_wait = False
        elif "WARPGROUP.DEPBAR.LE gsb0, 0x0" in line:
            full_wait = True
        elif re.search(r"\bBAR\.SYNC|\bEXIT\b", line):  # the epilogue: a new job starts after a named barrier
            full_wait = False
    return n, waits


def test_no_divergent_or_call_serialization(compiled):
    log, kernels = compiled
    assert len(kernels) == 36, sorted(kernels)
    bad = [l for l in log.splitlines() if re.search(r"\((C7520|C7510)\)", l)]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("name", sorted(PIPELINED))
def test_tap_products_issue_back_to_back(compiled, name):
    cin, cout, tail, mode = PIPELINED[name]
    n, waits = serialized_products(compiled[1][(cin, cout, F16F8, tail, mode)])
    assert n >= 2, f"{name}: {n} GMMA instructions"
    assert waits == 0, f"{name}: {waits} of {n} GMMAs wait for every earlier product"


@pytest.mark.parametrize("name", sorted(NOT_YET))
@pytest.mark.xfail(strict=True, reason="ptxas C7518: still serialized for Cout >= 32")
def test_wide_layers_issue_back_to_back(compiled, name):
    cin, cout, tail, mode = NOT_YET[name]
    n, waits = serialized_products(compiled[1][(cin, cout, F16F8, tail, mode)])
    assert n >= 2 and waits == 0
