"""The C-ABI library loads without a GPU and exports every symbol include/agp.h declares; the ctypes
mirror covers exactly that set.  No compute entry point is called here."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "agp.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(agp_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(ag):
    lib = ag._cabi.lib()
    names = _header_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), "libagp.so does not export %s" % n
    assert sorted(ag._cabi.SIGNATURES) == names, "ctypes mirror and agp.h disagree"


def test_version_and_host_only_helpers(ag):
    lib = ag._cabi.lib()
    assert b"sm_90a" in lib.agp_version()
    # 2D block-cyclic owner map (host-only): 2x4 grid
    owners = {(i, j): lib.agp_bc_owner(i, j, 2, 4) for i in range(6) for j in range(6)}
    assert owners[(0, 0)] == 0 and owners[(1, 0)] == 4 and owners[(0, 3)] == 3 and owners[(3, 5)] == 5
    nt = 16
    assert sum(lib.agp_bc_local_tiles(nt, r, 2, 4) for r in range(8)) == nt * (nt + 1) // 2


def test_no_cpu_fallback_without_gpu(ag):
    """Without a CUDA device the product path must fail loudly, never compute on the CPU."""
    import ctypes as C
    lib = ag._cabi.lib()
    h = C.c_void_p()
    rc = lib.agp_init(C.byref(h), 0, None)
    if rc == 0:  # running on a GPU box: nothing to assert here
        lib.agp_destroy(h)
        pytest.skip("GPU present")
    assert rc == ag._cabi.AGP_ERR_CUDA
    import numpy as np
    f = ag.GP(ag.SqExponentialKernel())
    with pytest.raises(ag.AGPError):
        ag.logpdf(f(np.linspace(0, 1, 5), 0.1), np.zeros(5))


def test_product_does_not_import_oracle():
    """oracle/ is test infrastructure: nothing under the product package may import it."""
    pkg = os.path.join(ROOT, "abstractgps.jl_b200")
    for dp, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dp, fn), errors="ignore").read()
                assert "oracle" not in txt.replace("# oracle-free", ""), fn


def test_header_is_plain_c_and_a_c_client_links(tmp_path):
    """include/agp.h is the boundary a C / Julia / Go host binds: it must compile as C99 (no C++-isms), and a C client
    (examples/c_abi_demo.c) must link against libagp.so; without a CUDA device the client reports the failure of
    agp_init and exits 2 -- no silent CPU path."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    inc = os.path.join(ROOT, "include")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c",
                        os.path.join(inc, "agp.h")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    exe = str(tmp_path / "c_abi_demo")
    libdir = os.path.join(ROOT, "abstractgps.jl_b200")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-I" + inc, os.path.join(ROOT, "examples", "c_abi_demo.c"), "-o", exe,
                        "-L" + libdir, "-l:libagp.so", "-lm", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode in (0, 2), (r.returncode, r.stdout, r.stderr)
    if r.returncode == 2:
        assert "agp_init" in r.stderr
    else:
        assert "logpdf" in r.stdout
