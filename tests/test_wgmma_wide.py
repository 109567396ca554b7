"""The wgmma convolutions of the 4-level U-Net (kernels_wgmma_wide.cu): a compile-time check, no GPU needed.

Every kernel must compile without spills and without the divergent-path (C7520) or function-call (C7510) serialization.
The kernels that ptxas still serializes are pinned exactly, so that a change in either direction shows up here:
C7518 (the wide layers, as in kernels_wgmma.cu) and C7511 (too few registers for the pipeline)."""
import os
import re
import subprocess

import pytest

from test_wgmma_issue import CUOBJDUMP, NVCC, ROOT, CSRC

pytestmark = pytest.mark.skipif(NVCC is None or CUOBJDUMP is None, reason="needs nvcc and cuobjdump")

F16, F16X2, F16F8 = 1, 2, 3
CONV, POOL, CONVT = 0, 1, 2
KERNELS = {(cin, cout, fmt, 0, mode) for fmt in (F16, F16X2, F16F8)
           for cin, cout, mode in ((64, 64, POOL), (128, 64, CONV), (128, 64, CONVT))}
C7518 = {(cin, cout, fmt, 0, mode) for fmt in (F16, F16X2, F16F8) for cin, cout, mode in ((64, 64, POOL), (128, 64, CONV))}
C7511 = {(128, 64, F16X2, 0, CONVT)}
NAME = re.compile(r"conv3_wgmma_kernelILi(\d+)ELi(\d+)ELi(\d)ELb(\d)ELi(\d)E")


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    out = tmp_path_factory.mktemp("wgmma_wide")
    res = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
                          "-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-cubin",
                          os.path.join(CSRC, "kernels_wgmma_wide.cu"), "-o", str(out / "wide.cubin")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return res.stdout + res.stderr


def _key(s):
    return tuple(int(g) for g in NAME.search(s).groups())


def test_kernels_and_spills(ptxas_log):
    spills, current = {}, None
    for line in ptxas_log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            current = _key(m.group(1)) if NAME.search(m.group(1)) else None
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            spills[current] = int(m.group(1)) + int(m.group(2))
    assert set(spills) == KERNELS, sorted(spills)
    assert all(v == 0 for v in spills.values()), spills


def test_serialization_is_pinned(ptxas_log):
    bad = [l for l in ptxas_log.splitlines() if re.search(r"\((C7520|C7510)\)", l)]
    assert not bad, "\n".join(bad)
    for code, expected in (("C7518", C7518), ("C7511", C7511)):
        got = {_key(l) for l in ptxas_log.splitlines() if f"({code})" in l}
        assert got == expected, (code, sorted(got))
