"""The exact model of the int8-slice update (tests/ozaki_exact_model.py) held to exact rational arithmetic on the CPU:
the slicing is error-free, the integer words stay inside the ranges the kernel's conversions need, and the modelled
result of C_old + sign * A B' is within the proven truncation bound of the exact value, at every instantiated slice
count and C type and at the K edges of the kernel (two chunks, the pair32 cutoff, the longest K the VFE stream uses).
tests/test_gpu_ozaki_exact.py then requires the kernel to equal this model bit for bit."""
from fractions import Fraction

import numpy as np
import pytest

import ozaki_exact_model as om

INSTANCES = [(4, "f64"), (5, "f64"), (6, "f64"), (7, "f64"), (8, "f64"), (3, "f32"), (4, "f32"), (5, "f32")]
KS = [64, 512, 576, 4096, 32768]


def _operands(rng, m, K, odt, lo=-30, hi=30):
    P = rng.standard_normal((m, K)) * np.ldexp(1.0, rng.integers(lo, hi, (m, 1)))
    return P.astype(odt).astype(np.float64)


def _model(A, B, C0, S, sign, c_is_float, pair32):
    """rectangular product of the rows of A and B, every entry owned"""
    M, N = A.shape[0], B.shape[0]
    ws = om.Workspace(S, A.shape[1], om.ceil128(M) + N).put(A).put(B, om.ceil128(M))
    cols = om.column_rows(N, om.tile_width(S), om.ceil128(M))
    flat = np.asarray(C0, dtype=np.float32 if c_is_float else np.float64).T.reshape(-1)   # column-major, ldc = M
    out = om.expected_update(ws, flat, M, M, N, sign, 0, cols, np.ones((M, N), bool), pair32, c_is_float)
    return out.reshape(N, M).T, ws


def _check_against_exact(got, A, B, C0, S, sign, c_is_float, extra=()):
    """sampled entries and the worst one (by an fp64 estimate) against the exact rational, under result_bound"""
    ea, _, _ = om.row_exponents(A)
    eb, _, _ = om.row_exponents(B)
    K = A.shape[1]
    approx = C0.astype(np.float64) + sign * (A @ B.T)
    scale = np.ldexp(1.0, ea[:, None] + eb[None, :]) * K
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = np.nan_to_num(np.abs(got.astype(np.float64) - approx) / scale, nan=0.0, posinf=0.0)
    worst = np.unravel_index(np.argmax(rel), got.shape)
    picks = {worst, (0, 0), (got.shape[0] - 1, got.shape[1] - 1), *extra}
    for i, j in picks:
        ex = om.exact_entry(C0[i, j], A[i], B[j], sign)
        err = abs(Fraction(float(got[i, j])) - ex)
        bnd = om.result_bound(S, ea[i], eb[j], K, got[i, j], c_is_float)
        assert err <= bnd, (i, j, float(err), float(bnd))


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("S,cdt", INSTANCES)
@pytest.mark.parametrize("odt", [np.float64, np.float32])
def test_model_is_within_the_exact_bound(S, cdt, K, odt):
    rng = np.random.default_rng(1000 * S + K % 997 + (odt == np.float32))
    m, n = (6, 5) if K >= 4096 else (12, 9)
    A, B = _operands(rng, m, K, odt), _operands(rng, n, K, odt)
    c_is_float = cdt == "f32"
    C0 = rng.standard_normal((m, n)) * np.ldexp(1.0, rng.integers(-20, 40, (m, n)))
    C0 = C0.astype(np.float32 if c_is_float else np.float64)
    sign = -1.0 if (S + K) % 2 else 1.0
    got, ws = _model(A, B, C0, S, sign, c_is_float, om.pair32_used(S, K))
    # the slicing is error-free: x 2^-e = sum_s q_s 2^-(6+7s) + r exactly, |q| <= 64, |r| <= 2^-7S
    _, _, rinv = om.row_exponents(A)
    q, r = om.slice_rows(A, S, rinv)
    assert np.abs(q).max() <= 64 and np.abs(r).max() <= 2.0 ** (-7 * S)
    for i, k in [(0, 0), (m - 1, K - 1), (m // 2, K // 3)]:
        lhs = Fraction(float(A[i, k])) * Fraction(float(rinv[i]))
        assert lhs == sum(Fraction(int(q[s, i, k]), 2 ** (6 + 7 * s)) for s in range(S)) + Fraction(float(r[i, k]))
    if S >= 5 and K <= 512:  # both drains give the same bits wherever the int32 pair form is used
        assert np.array_equal(got, _model(A, B, C0, S, sign, c_is_float, False)[0])
    _check_against_exact(got, A, B, C0, S, sign, c_is_float)


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("S", [3, 4, 5, 6, 7, 8])
def test_near_bound_digits(S, K):
    """digits 60..63 with one sign per row: the slicer returns them unchanged, the accumulators come within 12 % of
    their int32 bound (d+1) K 64^2 and the words of the 2^51 conversion limit at K = 32768, and the model stays exact
    up to its bound.  Above K = 512 the int32 pair form wraps on these inputs -- the launcher must not use it there."""
    rng = np.random.default_rng(S * 7 + K)
    m, n = 4, 3
    qa, qb = om.near_bound_digits(rng, S, m, K), om.near_bound_digits(rng, S, n, K)
    A, B = om.digits_to_values(qa), om.digits_to_values(qb)
    for P, qq in ((A, qa), (B, qb)):
        e, rscale, rinv = om.row_exponents(P)
        assert np.all(e == 0)
        q, r = om.slice_rows(P, S, rinv)
        assert np.array_equal(q, qq) and np.all(r == 0)
    acc = om.accumulators(qa, qb)
    for d in range(S):
        assert np.abs(acc[d]).min() >= (d + 1) * K * 60 * 60
    h, l = om.words(acc, False)
    hmax = sum((d + 1) * K * 4096 * 128 ** (3 - d) for d in range(min(S, 4)))
    lmax = sum((d + 1) * K * 4096 * 128 ** (S - 1 - d) for d in range(4, S))
    assert np.abs(h).min() >= 0.87 * hmax and np.abs(l).min() >= 0.87 * lmax
    assert hmax < 2 ** 51 and lmax < 2 ** 51 and (K < 32768 or S < 8 or lmax >= 2 ** 50)
    if S >= 5:
        same = np.array_equal(om.combine(acc, True), om.combine(acc, False))
        assert same == (K <= 576 or S == 5 and K < 1024)
    C0 = rng.random((m, n))
    for cdt in ("f64", "f32"):
        if (S, cdt) not in INSTANCES:
            continue
        c0 = C0.astype(np.float32 if cdt == "f32" else np.float64)
        got, _ = _model(A, B, c0, S, -1.0, cdt == "f32", om.pair32_used(S, K))
        _check_against_exact(got, A, B, c0, S, -1.0, cdt == "f32", extra=[(i, j) for i in range(m) for j in range(n)])


def test_row_exponents_at_the_edges_of_the_range():
    P = np.array([[1e-310, -3e-320, 0.0],          # subnormal only: e clamps to -1022, 2^1022 scales it exactly
                  [0.0, 0.0, 0.0],                 # zero row: e = 0
                  [2.0 ** 1000, -1.0, 2.0 ** -1000],
                  [np.nan, 1.0, 2.0],              # non-finite or >= 2^1023: rscale NaN, digits 0
                  [1.0, np.inf, 0.5],
                  [-np.inf, 1.0, 0.5],
                  [2.0 ** 1023, 1.0, 0.0],
                  [np.finfo(np.float64).max / 2.5, 1.0, 0.0]])
    e, rscale, rinv = om.row_exponents(P)
    assert list(e[:3]) == [-1022, 0, 1001] and e[7] == 1023
    assert np.all(np.isfinite(rinv)) and np.all(rinv[3:7] == 0)
    assert np.all(np.isnan(rscale[3:7])) and not np.isnan(rscale[7])
    q, r = om.slice_rows(P, 8, rinv)
    assert np.abs(q).max() <= 64 and np.all(q[:, 3:7] == 0)
    for k in range(3):  # the subnormal row is held to 2^-56 of 2^-1022: its digits are exact up to the residual
        ex = Fraction(float(P[0, k])) * 2 ** 1022
        assert abs(ex - sum(Fraction(int(q[s, 0, k]), 2 ** (6 + 7 * s)) for s in range(8))) <= Fraction(1, 2 ** 56)
    # a NaN or Inf row turns every entry it touches into NaN, as A row and as B column; the rest is unaffected
    B = np.ones((2, 3))
    got, _ = _model(P[[2, 3, 4]], B, np.zeros((3, 2)), 7, -1.0, False, True)
    assert np.all(np.isfinite(got[0])) and np.all(np.isnan(got[1:]))
    got, _ = _model(B, P[[2, 5]], np.zeros((2, 2)), 7, 1.0, False, True)
    assert np.all(np.isfinite(got[:, 0])) and np.all(np.isnan(got[:, 1]))


@pytest.mark.parametrize("cdt", ["f64", "f32"])
def test_subnormal_products_round_once(cdt):
    """C_old = 0 and row scales whose products land in the subnormal range of C: for fp64 C, v p falls below 2^-1022 and
    the fma's single rounding must be modelled exactly (and below 2^-1041 the scale product p itself flushes to 0, which
    the bound allows); one operand spans 2^-1000 .. 2^1000 (2^-150 .. 2^100 for fp32 C)"""
    rng = np.random.default_rng(5)
    K, S = 64, 5 if cdt == "f32" else 7
    ea = [-1000, -1010, -990, 1000, 0, -1060] if cdt == "f64" else [-130, -140, -120, 100, 0, -150]
    eb = [-60, -30, 0, -20] if cdt == "f64" else [-10, -5, 0, -20]
    A = rng.standard_normal((6, K)) * np.ldexp(1.0, np.array(ea)[:, None])
    B = rng.standard_normal((4, K)) * np.ldexp(1.0, np.array(eb)[:, None])
    c0 = np.zeros((6, 4), dtype=np.float32 if cdt == "f32" else np.float64)
    got, _ = _model(A, B, c0, S, 1.0, cdt == "f32", True)
    tiny = np.abs(got) < np.finfo(got.dtype).tiny
    assert tiny.sum() >= 6 and np.any(got[tiny] != 0)
    _check_against_exact(got, A, B, c0, S, 1.0, cdt == "f32", extra=[(i, j) for i in range(6) for j in range(4)])


def test_exact_fma_differs_from_two_roundings():
    """the reason for exact_fma: a product below 2^-1022 rounds before the add in numpy but not in an fma"""
    v, p, c = 1.5, 2.0 ** -1074, -(2.0 ** -1074)
    assert om.exact_fma(v, p, c) == 0.0 and v * p + c == 2.0 ** -1074


@pytest.mark.parametrize("BN", [32, 64])
def test_walk_masks(BN):
    """the closed-form lower walk and the strip table agree where both apply (identity map, a_off == b_off), and the
    table's block-cyclic column map sends each strip's columns to consecutive panel rows"""
    M, N = 640, 512
    assert np.array_equal(om.owned_lower(M, N, BN), om.owned_table(M, N, BN, 0, 0))
    rows = om.column_rows(N, BN, 256, stride=512, bw=128)
    assert list(rows[:3]) == [256, 257, 258] and rows[128] == 768 and rows[300] == 256 + 2 * 512 + 44
    own = om.owned_table(M, N, BN, 256, 128, stride=512, bw=128)
    assert not own[:128, 0].any() and own[128:, 0].all() and not own[:, 128:].all()
