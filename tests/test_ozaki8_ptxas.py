"""ptxas must pipeline the eight-bit update kernel (ozaki8_update_kernel) as it does the seven-bit ones: no wgmma
serialisation advisory (C75xx) and no spills, and the seven-bit instantiations are still the eight
ozaki_syrk_wgmma_kernel entries.  Compiles umma_ozaki.cu for sm_90a on the CPU; skips without nvcc."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "abstractgps.jl_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas8") / "umma_ozaki.o"
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "umma_ozaki.cu"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def test_eight_bit_kernel_pipelined_without_spills(report):
    assert not [l for l in report.splitlines() if re.search(r"\(C75\d\d\)", l) and "ozaki8_update_kernel" in l]
    entries = re.split(r"Compiling entry function '", report)[1:]
    mine = [e for e in entries if e.split("'")[0].endswith("ozaki8_update_kernelENS_10OzTileArgsEliii")]
    assert len(mine) == 1
    spill = [l for l in mine[0].splitlines() if "spill" in l]
    assert spill and all("0 bytes spill stores, 0 bytes spill loads" in l for l in spill), spill
    assert sum(1 for e in entries if "ozaki_syrk_wgmma_kernel" in e.split("'")[0]) == 8
