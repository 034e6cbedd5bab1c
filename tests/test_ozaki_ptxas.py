"""ptxas must pipeline the int8-slice trailing kernel: no instantiation of ozaki_syrk_wgmma_kernel may have its wgmma issue
serialised (ptxas advisory C7511, "insufficient register resources for the wgmma pipeline") or spill to local memory.
Either costs a large share of the kernel's tensor throughput without changing a result, so only the compiler's report
shows it.  Compiles umma_ozaki.cu for sm_90a on the CPU; skips without nvcc."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "abstractgps.jl_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "umma_ozaki.o"
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "umma_ozaki.cu"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def _entries(report):
    """{mangled kernel name: its ptxas lines} for every entry function"""
    out, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur is not None:
            out[cur].append(line)
    return out


def test_trailing_kernel_wgmma_not_serialised(ptxas_report):
    bad = [l for l in ptxas_report.splitlines() if re.search(r"\(C75\d\d\)", l) and "ozaki_syrk_wgmma_kernel" in l]
    assert not bad, "\n".join(bad)


def test_trailing_kernel_no_spills(ptxas_report):
    kernels = {k: v for k, v in _entries(ptxas_report).items() if "ozaki_syrk_wgmma_kernel" in k}
    assert len(kernels) == 8  # fp64 C: S = 4..8; fp32 C: S = 3..5
    for name, lines in kernels.items():
        spill = [l for l in lines if "spill" in l]
        assert spill, name
        assert all("0 bytes spill stores, 0 bytes spill loads" in l for l in spill), (name, spill)
