"""The tile GEMM (csrc/gemm.cu) bit for bit against its exact model (tests/gemm_exact_model.py), through agp_debug_gemm:
every kernel the contract lets a product select (fp64 DMMA: 4 storage orders, C == A and C == B; fp32 FFMA), M, N and K
at and around the tile edges, alpha = +-1, beta in {0, 1}, lower_only, trmm_lower with finite storage above the
diagonal, and the block-cyclic column maps of the distributed trailing update.  Every element of an operand buffer
outside op(A) / op(B) is NaN, so reading one poisons an owned entry; every C element the kernel does not own, padding and
a tail past the buffer included, must be unchanged bit for bit.  Each call is exactly one launch.  Products that break
the contract are refused before anything is launched."""
import ctypes as C
from dataclasses import replace

import numpy as np
import pytest

import gemm_exact_model as gm

pytestmark = pytest.mark.gpu


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def _call(ag, g, A, B, Cbuf):
    """one agp_debug_gemm on device copies of the buffers; returns (status, launches, C buffer after the call)"""
    import torch
    from agp_b200 import _cabi
    eng = ag.engine()
    Cd = _dev(Cbuf)
    Ad = Cd if A is Cbuf else _dev(A)
    Bd = Cd if B is Cbuf else _dev(B)
    torch.cuda.synchronize()
    dtype = _cabi.AGP_F64 if g.dtype == np.float64 else _cabi.AGP_F32
    n0 = eng.L.agp_launch_count(eng.h)
    rc = eng.L.agp_debug_gemm(eng.h, dtype, _ptr(Ad, g.a_misalign), g.a_kmajor, g.lda, _ptr(Bd, g.b_misalign), g.b_kmajor,
                              g.ldb, _ptr(Cd, g.c_misalign), g.ldc, g.M, g.N, g.K, g.alpha_neg, g.beta_one, g.lower_only,
                              g.trmm_lower, g.stride, g.width, g.b_off)
    return rc, eng.L.agp_launch_count(eng.h) - n0, Cd.cpu().numpy()


def _same_bits(got, want, what=""):
    ut = np.uint64 if got.dtype == np.float64 else np.uint32
    bad = np.nonzero(got.view(ut) != want.view(ut))[0]
    assert bad.size == 0, "%s: %d elements differ, first at %s: got %r want %r" % (what, bad.size, bad[:8], got[bad[:4]],
                                                                                 want[bad[:4]])


def _check(ag, g, seed):
    assert gm.contract_ok(g), g
    A, B, Cbuf = gm.make_buffers(g, np.random.default_rng(seed))
    want, own = gm.expected(g, A, B, Cbuf)
    rc, launches, got = _call(ag, g, A, B, Cbuf)
    ag.engine().check(rc)
    assert launches == (1 if g.M > 0 and g.N > 0 else 0), (launches, g)
    _same_bits(got, want, "%s %s" % (gm.kernel_name(g), g))
    assert not np.isnan(got[gm.c_index(g)][own]).any()
    return own


@pytest.mark.parametrize("inst", gm.INSTANTIATIONS, ids=lambda t: "%s-a%d-b%d-%s" % (np.dtype(t[0]).name, t[1], t[2],
                                                                                        t[3] or "sep"))
def test_instantiation_shapes(ag, inst):
    for i, g in enumerate(gm.instantiation_cases(*inst) + gm.pinning_cases(*inst)):
        _check(ag, g, 1000 * gm.INSTANTIATIONS.index(inst) + i)


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_column_maps(ag, dt):
    for i, g in enumerate(gm.map_cases(dt)):
        own = _check(ag, g, 77 + i)
        assert own.any() and (own.all() or g.lower_only)


def test_trailing_update_fallback_map(ag):
    """the arguments trailing_update passes the GEMM when row0 != col0: C = L[row0.., col0..], A = B = L[row0.., kcol0..]
    (B from row0), and the map shifts column n to panel row col0 - row0 + n, stride 128"""
    row0, col0, K, lda = 256, 640, 128, 1408
    M, N = lda - row0, 384
    g = gm.Gemm(np.float64, M, N, K, lda=lda, ldb=lda, ldc=lda, alpha_neg=1, beta_one=1, lower_only=1, stride=128,
                b_off=col0 - row0)
    assert gm.contract_ok(g)
    own = _check(ag, g, 5)
    assert own.any() and not own.all()


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_real_values_within_the_error_bound(ag, dt):
    """random normal data: |C - ref| <= gamma_(K+1) (|c| + |A||B|) against an extended-precision reference"""
    rng = np.random.default_rng(11)
    u = np.finfo(dt).eps / 2
    for M, N, K, akm, bkm in ((300, 300, 1030 if dt == np.float64 else 1028, 0, 1), (129, 65, 130 if dt == np.float64 else 132, 1, 0)):
        M = M if dt == np.float64 else M // 4 * 4
        g = gm.with_lds(gm.Gemm(dt, M, N, K, a_kmajor=akm, b_kmajor=bkm, alpha_neg=1, beta_one=1))
        A = np.full(g.lda * (M if akm else K), np.nan, dtype=dt)
        B = np.full(g.ldb * (N if bkm else K), np.nan, dtype=dt)
        Cbuf = np.full(g.ldc * N, np.nan, dtype=dt)
        a, b, c = (rng.standard_normal(s).astype(dt) for s in ((M, K), (K, N), (M, N)))
        m, k, n = np.arange(M)[:, None], np.arange(K)[None, :], np.arange(N)[None, :]
        A[(k + m * g.lda) if akm else (m + k * g.lda)] = a
        B[(k.T + n * g.ldb) if bkm else (n + k.T * g.ldb)] = b
        Cbuf[gm.c_index(g)] = c
        rc, _, got = _call(ag, g, A, B, Cbuf)
        ag.engine().check(rc)
        ld = np.longdouble
        ref = c.astype(ld) - a.astype(ld) @ b.astype(ld)
        gam = (K + 1) * u / (1 - (K + 1) * u)
        bound = gam * (np.abs(c).astype(ld) + np.abs(a).astype(ld) @ np.abs(b).astype(ld))
        err = np.abs(got[gm.c_index(g)].astype(ld) - ref)
        assert np.all(err <= bound), float((err / bound).max())
        assert float((err / bound).max()) > 1e-6  # the comparison sees the kernel's rounding, not a copy of the reference


def _violations():
    """(reason, product): each breaks exactly one clause of the contract; the buffers are valid for the product
    without that clause"""
    f64 = gm.with_lds(gm.Gemm(np.float64, 128, 128, 64, a_kmajor=1, b_kmajor=0, beta_one=1))
    f32 = gm.with_lds(gm.Gemm(np.float32, 128, 128, 64, a_kmajor=0, b_kmajor=1, beta_one=1))
    ca = gm.with_lds(gm.Gemm(np.float64, 128, 128, 128, alias="A"))
    cb = gm.with_lds(gm.Gemm(np.float64, 128, 128, 128, b_kmajor=1, alias="B"))
    mp = gm.with_lds(gm.Gemm(np.float64, 512, 256, 128, stride=512, width=128, b_off=0))
    return [
        ("fp64 A misaligned", replace(f64, a_misalign=1)),
        ("fp64 B misaligned", replace(f64, b_misalign=1)),
        ("fp64 odd lda", replace(f64, lda=f64.lda + 1)),
        ("fp64 odd ldb", replace(f64, ldb=f64.ldb + 1)),
        ("fp64 odd K, A K-major", replace(f64, K=63)),
        ("fp64 lda below K", replace(f64, lda=62)),
        ("fp64 ldb below N", replace(f64, ldb=126)),
        ("fp64 ldc below M", replace(f64, ldc=126)),
        ("fp32 A misaligned", replace(f32, a_misalign=2)),
        ("fp32 C misaligned", replace(f32, c_misalign=1)),
        ("fp32 lda % 4", replace(f32, lda=f32.lda + 2)),
        ("fp32 ldc % 4", replace(f32, ldc=f32.ldc + 2)),
        ("fp32 K % 4, B K-major", replace(f32, K=62)),
        ("fp32 M % 4", replace(f32, M=126)),
        ("C == A, A K-major", replace(ca, a_kmajor=1, lda=128)),
        ("C == A, ldc != lda", replace(ca, ldc=ca.lda - 2)),
        ("C == A, N > 128", replace(ca, N=130)),
        ("C == B, B MN-major", replace(cb, b_kmajor=0)),
        ("C == B, ldc != ldb", replace(cb, ldc=cb.ldb - 2)),
        ("C == B, M > 128", replace(cb, M=130)),
        ("C == B, column map", replace(cb, stride=256, N=128)),
        ("map width not a tile multiple", replace(mp, width=96)),
        ("map negative offset", replace(mp, b_off=-128)),
        ("map shift misaligned, B MN-major", replace(mp, b_off=1, ldb=mp.ldb + 2)),
        ("map past ldb", replace(mp, b_off=256)),
    ]


@pytest.mark.parametrize("reason,g", _violations(), ids=[r for r, _ in _violations()])
def test_contract_violations_are_refused(ag, reason, g):
    """never launched: the status is AGP_ERR_INVALID, the launch counter does not move and C is untouched"""
    from agp_b200 import _cabi
    assert not gm.contract_ok(g), reason
    valid = replace(g, a_misalign=0, b_misalign=0, c_misalign=0, K=max(g.K, 0))
    rows = max(valid.lda, valid.ldb, valid.ldc, 1)
    cols = max(valid.M, valid.N, valid.K, gm.highest_b_column(valid) + 1) + 4
    size = rows * cols + 64  # room for every element any clause-free reading of the arguments could address
    rng = np.random.default_rng(3)
    A = rng.standard_normal(size).astype(g.dtype)
    B = rng.standard_normal(size).astype(g.dtype)
    Cbuf = rng.standard_normal(size).astype(g.dtype)
    if g.alias == "A":
        A = Cbuf
    if g.alias == "B":
        B = Cbuf
    rc, launches, got = _call(ag, g, A, B, Cbuf)
    assert rc == _cabi.AGP_ERR_INVALID, reason
    assert launches == 0
    _same_bits(got, Cbuf, reason)
