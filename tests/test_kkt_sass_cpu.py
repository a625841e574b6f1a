"""CPU check of the instructions the KKT factorisation runs on the fp64 tensor core (cuobjdump -sass of the built
libchd.so): the panel and the trailing updates of chd_k_kkt and chd_k_kkt_gwin use Hopper's DMMA.16x8x8, which runs
at twice the rate of the Ampere shape DMMA.8x8x4; only warp 0's single next-diagonal-tile update keeps a pair of
DMMA.8x8x4.  The fp64 probe behind bench.py's roofline denominator issues the same DMMA.16x8x8."""
import collections
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "contact-human-dynamics_b200", "libchd.so")
KERNELS = {"kkt": "_Z9chd_k_kkt6ChdDev", "gwin": "_Z14chd_k_kkt_gwin6ChdDev", "peak": "_Z15chd_k_fp64_peakiiPd"}
SINGLE_TILE_MAX = 4   # chd_tile_sub_xyT: two DMMA.8x8x4, room for the compiler to duplicate them once


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


@pytest.fixture(scope="module")
def dmma():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump is not available")
    if not os.path.exists(LIB):
        pytest.skip("libchd.so is not built")
    sass = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    counts = collections.defaultdict(collections.Counter)
    fn = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"\bDMMA\.(\w+)", line)
        if m and fn is not None:
            counts[fn][m.group(1)] += 1
    return counts


@pytest.mark.parametrize("kernel", ["kkt", "gwin"])
def test_kkt_factorisation_uses_dmma_16x8x8(dmma, kernel):
    c = dmma[KERNELS[kernel]]
    assert c["16x8x8"] > 0, dict(c)
    assert c["8x8x4"] <= SINGLE_TILE_MAX, dict(c)


def test_fp64_probe_issues_dmma_16x8x8(dmma):
    c = dmma[KERNELS["peak"]]
    assert c["16x8x8"] > 0 and c["8x8x4"] == 0, dict(c)
