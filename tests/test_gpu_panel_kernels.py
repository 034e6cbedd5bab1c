"""One step of the blocked Cholesky (csrc/potrf.cu and the panel GEMM), through agp_debug_panel, on every route: fp64
factor-only kernel + substitution TRSM, fp64 factor-only kernel + strip inverse + in-place GEMM, the fused fp64 kernel +
GEMM, and the fused fp32 kernel + GEMM.

Bounds (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Thm 10.3 for the factor, 8.5 for the
triangular solves and inverse; u the unit roundoff, gamma_n = n u / (1 - n u)), with a factor 2 for the refined
approximate rsqrt of the diagonal:
    |A - L L'| <= 2 gamma_129 |L||L'|,  |B - X L'| <= 2 gamma_128 |X||L'| (substitution),
    |X - B D'| <= gamma_128 |B||D'| (inverse routes: X is one GEMM with D = Dinv),  |L D - I| <= 2 gamma_128 |L||D|.
Residuals are evaluated in x86 extended precision, whose own error (2^-64 per operation) is more than 2^10 times below
the fp64 bounds.  The upper triangles of L and Dinv must be exactly zero, logdet[blk] must match sum log diag(L0) for
A = L0 L0' with an integer L0, rows past the panel and storage outside the block must be untouched, and info must equal
LAPACK's potrf on the same block (offset by blk * 128) at every tested first failing pivot.  A positive subnormal pivot
is factored, as LAPACK factors it, rather than turned into a non-finite factor with info = 0."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg.lapack as lapack

pytestmark = pytest.mark.gpu

T = 128
SENTINEL = -7.25
ROUTES = [("f64", 0), ("f64", 1), ("f64", 2), ("f32", 2)]  # (dtype, AGP_PANEL_*)
IDS = ["f64-subst", "f64-inverse-gemm", "f64-fused", "f32-fused"]


def _dt(name):
    return np.float64 if name == "f64" else np.float32


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _run(ag, dname, route, Ablk, panel, blk=0, info0=0, extra_rows=5, extra_cols=2):
    """factor Ablk (128 x 128, lower triangle used) with `panel` (rows_below x 128) below it; the column-major buffer has
    extra rows and columns of SENTINEL around them.  Returns (status, L, X, Dinv, logdet[blk], info, buffer, Dinv buffer)"""
    import torch
    from agp_b200 import _cabi
    dt = _dt(dname)
    rb = panel.shape[0]
    lda = -(-(T + rb + extra_rows) // 4) * 4
    buf = np.full((T + extra_cols, lda), SENTINEL, dtype=dt)  # buf[c, r] = element (r, c)
    buf[:T, :T] = Ablk.T
    buf[:T, T:T + rb] = panel.T
    Dinv = np.full(T * T + 16, SENTINEL, dtype=dt)
    logdet = np.full(blk + 2, SENTINEL)
    info = np.array([info0], dtype=np.int32)
    bd, dd, ld, idv = _dev(buf.ravel()), _dev(Dinv), _dev(logdet), _dev(info)
    torch.cuda.synchronize()
    eng = ag.engine()
    p = lambda t: C.c_void_p(t.data_ptr())
    rc = eng.L.agp_debug_panel(eng.h, _cabi.AGP_F64 if dt == np.float64 else _cabi.AGP_F32, route, p(bd), lda, rb, blk,
                               p(dd), p(ld), p(idv))
    out = bd.cpu().numpy().reshape(T + extra_cols, lda)
    dv = dd.cpu().numpy()
    return (rc, out[:T, :T].T.copy(), out[:T, T:T + rb].T.copy(), dv[:T * T].reshape(T, T).T.copy(),
            ld.cpu().numpy(), int(idv.cpu().numpy()[0]), (buf, out), (Dinv, dv))


def _gamma(n, dt):
    u = np.finfo(dt).eps / 2
    return n * u / (1 - n * u)


def _le(lhs, rhs, what):
    ok = lhs <= rhs
    assert ok.all(), "%s: %d entries over the bound, worst ratio %.3g" % (what, (~ok).sum(), float(np.max(lhs / np.where(rhs > 0, rhs, 1))))


def _int_factor(rng, dt):
    """integer, diagonally dominant lower-triangular L0 (cond(A) ~ 1e3); A = L0 L0' is exact in dt"""
    hi = 2 if dt == np.float64 else 1
    L0 = np.tril(rng.integers(-hi, hi + 1, (T, T))).astype(np.float64)
    np.fill_diagonal(L0, np.abs(L0).sum(1) - np.abs(np.diag(L0)) + rng.integers(1, 8, T))
    A = L0 @ L0.T
    assert np.abs(A).max() < 2 ** 20
    return L0, A


def _se_block(rng, cond):
    """squared-exponential Gram block of 128 sorted points with a jitter that sets cond(A) near `cond`"""
    x = np.sort(rng.random(T)) * 4.0
    K = np.exp(-0.5 * (x[:, None] - x[None, :]) ** 2 / 0.6 ** 2)
    w = np.linalg.eigvalsh(K)
    return K + np.eye(T) * max(w[-1] / cond, 0.0)


def _check_factor(dname, route, A, panel, res, what):
    rc, L, X, D, logdet, info, (buf0, buf1), (d0, d1) = res
    dt = _dt(dname)
    assert rc == 0 and info == 0, (rc, info, what)
    ld = np.longdouble
    assert np.all(np.triu(L, 1) == 0) and np.all(np.triu(D, 1) == 0), what
    assert np.isfinite(L).all() and np.isfinite(D).all() and np.isfinite(X).all(), what
    Ll, Dl, Al = L.astype(ld), D.astype(ld), np.tril(A).astype(ld)
    absL = np.abs(Ll)
    _le(np.tril(np.abs(Al - Ll @ Ll.T)), 2 * _gamma(T + 1, dt) * np.tril(absL @ absL.T), what + " factor")
    _le(np.abs(Ll @ Dl - np.eye(T, dtype=ld)), 2 * _gamma(T, dt) * (absL @ np.abs(Dl)), what + " inverse")
    if panel.shape[0]:
        rows = np.unique(np.r_[np.arange(0, panel.shape[0], max(1, panel.shape[0] // 512)), panel.shape[0] - 1])
        Bl, Xl = panel[rows].astype(ld), X[rows].astype(ld)
        if route == 0:
            _le(np.abs(Bl - Xl @ Ll.T), 2 * _gamma(T, dt) * (np.abs(Xl) @ absL.T), what + " panel")
        else:
            _le(np.abs(Xl - Bl @ Dl.T), _gamma(T, dt) * (np.abs(Bl) @ np.abs(Dl.T)), what + " panel")
    # nothing outside the block, the panel and Dinv written
    rb = panel.shape[0]
    keep = np.ones(buf0.shape, bool)
    keep[:T, :T + rb] = False
    assert np.array_equal(buf0[keep].view(np.uint8), buf1[keep].view(np.uint8)), what + " storage outside"
    assert np.array_equal(d0[T * T:].view(np.uint8), d1[T * T:].view(np.uint8)), what + " past Dinv"


@pytest.mark.parametrize("dname,route", ROUTES, ids=IDS)
@pytest.mark.parametrize("rows_below", [0, 1, 31, 32, 33, 1000, 8192])
def test_known_factor(ag, dname, route, rows_below):
    rng = np.random.default_rng(rows_below + 10 * route)
    dt = _dt(dname)
    L0, A = _int_factor(rng, dt)
    panel = rng.standard_normal((rows_below, T)).astype(dt)
    blk = 3 if rows_below % 2 else 0
    res = _run(ag, dname, route, A.astype(dt), panel, blk=blk)
    if dt == np.float32 and rows_below % 4:  # the fp32 panel GEMM needs M % 4 == 0: refused before anything runs
        from agp_b200 import _cabi
        (buf0, buf1), (d0, d1) = res[6], res[7]
        assert res[0] == _cabi.AGP_ERR_INVALID and res[5] == 0
        assert np.array_equal(buf0.view(np.uint8), buf1.view(np.uint8)) and np.array_equal(d0.view(np.uint8), d1.view(np.uint8))
        return
    _check_factor(dname, route, A, panel, res, "rows_below=%d" % rows_below)
    logdet = res[4]
    want = float(np.sum(np.log(np.diag(L0))))
    assert abs(logdet[blk] - want) <= 8 * T * np.finfo(dt).eps * max(1.0, abs(want)), (logdet[blk], want)
    assert np.all(np.delete(logdet, blk) == SENTINEL)
    tol = 64 * T * np.finfo(dt).eps
    assert np.allclose(res[1], L0, rtol=0, atol=tol * np.abs(L0).max() * 8)


@pytest.mark.parametrize("dname,route", ROUTES, ids=IDS)
@pytest.mark.parametrize("cond", [1e4, 1e10])
def test_ill_conditioned_se_blocks(ag, dname, route, cond):
    dt = _dt(dname)
    if dt == np.float32 and cond > 1e6:
        cond = 1e5  # beyond 1/u the fp32 block is not numerically positive definite
    rng = np.random.default_rng(int(np.log10(cond)))
    A = _se_block(rng, cond).astype(dt).astype(np.float64)
    panel = rng.standard_normal((300, T)).astype(dt)
    _check_factor(dname, route, A, panel, _run(ag, dname, route, A.astype(dt), panel), "cond=%g" % cond)


PIVOTS = [1, 2, 7, 8, 9, 16, 17, 64, 121, 127, 128]


@pytest.mark.parametrize("dname,route", ROUTES, ids=IDS)
def test_info_matches_lapack(ag, dname, route):
    """first failing pivot j: made clearly negative (A_jj lowered by L0_jj^2 + 1000), or NaN, or -Inf; info =
    blk * 128 + j as LAPACK reports it, an info already set is kept, a positive definite block leaves 0"""
    dt = _dt(dname)
    potrf = lapack.dpotrf if dt == np.float64 else lapack.spotrf
    rng = np.random.default_rng(99)
    L0, A0 = _int_factor(rng, dt)
    panel = rng.standard_normal((40, T)).astype(dt)
    for i, j in enumerate(PIVOTS):
        for kind in ("neg",) + (("nan", "-inf") if j in (1, 8, 9, 128) else ()):
            A = A0.copy()
            A[j - 1, j - 1] = {"neg": A0[j - 1, j - 1] - L0[j - 1, j - 1] ** 2 - 1000.0, "nan": np.nan, "-inf": -np.inf}[kind]
            # reference LAPACK's potrf2 reports a NaN pivot (DISNAN); optimised builds may not, so NaN is held to j
            lap = j if kind == "nan" else potrf(A.astype(dt), lower=1, clean=0)[1]
            assert lap == j, (j, kind, lap)
            for blk in (0, 3):
                got = _run(ag, dname, route, A.astype(dt), panel, blk=blk)
                assert got[0] == 0
                assert got[5] == blk * T + lap, (j, kind, blk, got[5])
    A = A0.copy()
    A[8, 8] = -5.0
    assert _run(ag, dname, route, A.astype(dt), panel, info0=7)[5] == 7
    assert _run(ag, dname, route, A0.astype(dt), panel)[5] == 0


@pytest.mark.parametrize("dname,route", ROUTES, ids=IDS)
@pytest.mark.parametrize("j", [0, 9, 127])
def test_subnormal_pivot(ag, dname, route, j):
    """a positive subnormal pivot is factored as LAPACK factors it: finite, info = 0, L_jj = sqrt(p)"""
    dt = _dt(dname)
    p = 1e-310 if dt == np.float64 else 1e-40
    rng = np.random.default_rng(j)
    L0, A = _int_factor(rng, dt)
    A[j, :] = 0.0
    A[:, j] = 0.0
    A[j, j] = p
    Ad = A.astype(dt)
    Lref, lap = (lapack.dpotrf if dt == np.float64 else lapack.spotrf)(Ad, lower=1, clean=1)
    assert lap == 0
    panel = rng.standard_normal((32, T)).astype(dt)
    panel[:, j] = 0.0
    rc, L, X, D, logdet, info, _, _ = _run(ag, dname, route, Ad, panel)
    assert rc == 0 and info == 0
    assert np.isfinite(L).all() and np.isfinite(D).all() and np.isfinite(X).all() and np.isfinite(logdet[0])
    assert abs(float(L[j, j]) - np.sqrt(float(dt(p)))) <= 4 * np.finfo(dt).eps * np.sqrt(float(dt(p)))
    assert abs(float(D[j, j]) * float(L[j, j]) - 1.0) <= 8 * np.finfo(dt).eps
    assert np.allclose(L, Lref, rtol=0, atol=64 * T * np.finfo(dt).eps * np.abs(Lref).max())
