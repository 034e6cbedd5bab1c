"""Static checks of the composite-kernel plumbing that need no GPU: the Julia shim's structs match include/agp.h and the
ctypes mirror field for field, and no instantiation of the composite Gram and gradient kernels spills registers or uses a
stack frame (ptxas -v on gram.cu and grad.cu for sm_90a; skips without nvcc)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "abstractgps.jl_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _kind_c(t):
    t = t.strip()
    return "ptr" if "*" in t else {"int32_t": "i32", "double": "f64"}[t]


def _kind_j(t):
    return "ptr" if t.startswith("Ptr") else {"Int32": "i32", "Float64": "f64"}[t]


def _kind_ct(t):
    if t in (C.c_void_p,) or hasattr(t, "contents") or t.__name__.startswith("LP_"):
        return "ptr"
    return {C.c_int32: "i32", C.c_double: "f64"}[t]


def _c_struct(src, name):
    end = re.search(r"\}\s*%s;" % name, src).start()
    body = src[src.rindex("typedef struct {", 0, end) + len("typedef struct {"):end]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        m = re.match(r"(const\s+)?([\w]+\s*\**)\s*(.*)", decl)
        base = m.group(2).replace(" ", "")
        for v in m.group(3).split(","):
            v = v.strip()
            ptr = base.endswith("*") or v.startswith("*")
            out.append((v.lstrip("*").strip(), "ptr" if ptr else _kind_c(base)))
    return out


def _j_struct(src, name):
    m = re.search(r"struct %s;(.*?)end" % name, src)
    return [(f.split("::")[0].strip(), _kind_j(f.split("::")[1].strip())) for f in m.group(1).split(";") if f.strip()]


@pytest.mark.parametrize("c_name,j_name,py_name", [("agp_kernel", "AgpKernel", "agp_kernel"),
                                                   ("agp_kernel_factor", "AgpKernelFactor", "agp_kernel_factor"),
                                                   ("agp_kernel_composite", "AgpKernelComposite", "agp_kernel_composite")])
def test_julia_and_ctypes_structs_match_header(ag, c_name, j_name, py_name):
    h = open(os.path.join(ROOT, "include", "agp.h")).read()
    j = open(os.path.join(ROOT, "julia", "AGPBlackwell.jl")).read()
    c = _c_struct(h, c_name)
    assert _j_struct(j, j_name) == c
    assert [(n, _kind_ct(t)) for n, t in getattr(ag._cabi, py_name)._fields_] == c


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out = ""
    for src in ("gram.cu", "grad.cu"):
        obj = tmp_path_factory.mktemp("ptxas") / (src + ".o")
        cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
               "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
        out += r.stdout + r.stderr
    return out


def test_composite_kernels_do_not_spill(ptxas_report):
    entries, cur = {}, None
    for line in ptxas_report.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
            entries[cur] = []
        elif cur is not None:
            entries[cur].append(line)
    gram = [k for k in entries if "composite_gram_kernel" in k]
    grad = [k for k in entries if "composite_grad_reduce_kernel" in k]
    assert len(gram) == 16 and len(grad) == 16  # 1..8 accumulators x fp32 / fp64
    for name in gram + grad:
        frame = [l for l in entries[name] if "stack frame" in l]
        assert frame, name
        assert all("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in l for l in frame), (name, frame)


def test_julia_claim_and_limits_agree_with_the_python_mirror(ag):
    """the Julia shim claims the same families, builds the same descriptor family codes and applies the same limits
    (terms and factors in all) as the Python mirror"""
    j = open(os.path.join(ROOT, "julia", "AGPBlackwell.jl")).read()
    cabi = ag._cabi
    assert int(re.search(r"const AGP_COMPOSITE_MAX = (\d+)", j).group(1)) == cabi.AGP_COMPOSITE_MAX
    assert int(re.search(r"const AGP_COMPOSITE = Int32\((\d+)\)", j).group(1)) == cabi.AGP_COMPOSITE
    fam = {m.group(1): int(m.group(2)) for m in re.finditer(r"family\(::(\w+)\) = Int32\((\d+)\)", j)}
    assert fam == {"SqExponentialKernel": 0, "Matern12Kernel": 1, "Matern32Kernel": 2, "Matern52Kernel": 3, "LinearKernel": 4,
                   "RationalQuadraticKernel": cabi.AGP_RQ, "PeriodicKernel": cabi.AGP_PERIODIC, "WhiteKernel": cabi.AGP_WHITE,
                   "ConstantKernel": cabi.AGP_CONSTANT}
    only = set(re.search(r"const FactorOnly = Union\{([^}]*)\}", j).group(1).replace(" ", "").split(","))
    assert only == {"RationalQuadraticKernel", "PeriodicKernel", "WhiteKernel", "ConstantKernel"}
    for name in only:  # the Python mirror builds the same factor families under the same names
        assert callable(getattr(ag, name))
    assert re.search(r"composite_ok\(k::Union\{KernelSum,KernelProduct\}\) = all\(composite_ok, k\.kernels\)", j)
    lim = re.search(r"within_limits\(terms\) = (.*)", j).group(1)
    assert "length(terms) <= AGP_COMPOSITE_MAX" in lim and "sum(t -> length(t[2]), terms) <= AGP_COMPOSITE_MAX" in lim
    # Python: the same limits on the same flattening (terms > 8 or factors > 8 raise)
    three = ag.SqExponentialKernel() + ag.Matern12Kernel() + ag.Matern32Kernel()
    with pytest.raises(ag.AGPError):
        ag.api._Flat(three * three, 1)
    fl = ag.api._Flat(three * ag.WhiteKernel() + ag.ConstantKernel(), 1)
    assert len(fl.terms) == 4 and sum(len(f) for _, f in fl.terms) == 7
    # the exact-path methods claim composites; the VFE methods keep the single-kernel predicate (they fall through)
    for sig in ("logpdf(fx::DevFiniteGP{T}, Y::AbstractVecOrMat{<:Real}) where {T} =\n    claimed(fx.f)",
                "posterior(fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T} =\n    claimed(fx.f)",
                "claimed(fx.f) || return invoke(Random.rand"):
        assert sig in j, sig
    assert "supported(fx.f) ? sparse_objectives" in j and "claimed(fx.f) ? sparse_objectives" not in j
