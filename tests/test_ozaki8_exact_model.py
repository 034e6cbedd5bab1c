"""The exact model of the eight-bit format (tests/ozaki8_exact_model.py) held to exact rational arithmetic on the CPU: the
split is exact and its digits stay in the ranges the kernel stores as int8, the int32 diagonals and the int64 words stay
inside the ranges the kernel's conversions need up to K = 16384 (and the accumulator bound fails above it), and the
modelled C_old + sign * A B' is within the per-term bound of about 2^-43.4 2^(e_i+e_j) K of the exact value.
tests/test_gpu_ozaki8_exact.py then requires the kernel to equal this model bit for bit."""
from fractions import Fraction
import math

import numpy as np
import pytest

import ozaki_exact_model as om
import ozaki8_exact_model as o8

KS = [64, 512, 1024, 16384]


def _operands(rng, m, K, lo=-30, hi=30):
    return rng.standard_normal((m, K)) * np.ldexp(1.0, rng.integers(lo, hi, (m, 1)))


def _model(A, B, C0, sign):
    """rectangular product of the rows of A and B, every entry owned"""
    M, N = A.shape[0], B.shape[0]
    ws = o8.Workspace(A.shape[1], om.ceil128(M) + N).put(A).put(B, om.ceil128(M))
    cols = om.column_rows(N, om.tile_width(6), om.ceil128(M))
    flat = np.asarray(C0, dtype=np.float64).T.reshape(-1)
    out = o8.expected_update(ws, flat, M, M, N, sign, 0, cols, np.ones((M, N), bool))
    return out.reshape(N, M).T


def test_split_is_exact_and_digits_fit_int8():
    """X = rint(y 2^46) is rebuilt exactly from its digits; |q_0| <= 64, tails in [-128, 127], |y - X 2^-46| <= 2^-47,
    on random rows and on the values that push the leading digit to its extremes"""
    rng = np.random.default_rng(5)
    P = _operands(rng, 40, 256)
    edge = np.array([[1 - 2.0 ** -53, -(1 - 2.0 ** -53), 0.5, -0.5, 2.0 ** -47, -2.0 ** -47, 2.0 ** -48, 0.0,
                      (2 ** 46 - 2 ** 39 - 1) * 2.0 ** -46, -(2 ** 46 - 2 ** 39 - 1) * 2.0 ** -46] * 4])
    P = np.vstack([P, np.hstack([edge, np.zeros((1, 256 - edge.shape[1]))])])
    _, _, rinv = om.row_exponents(P)
    q = o8.slice_rows(P, rinv)
    assert np.abs(q[0]).max() <= o8.Q0_MAX and np.abs(q[0]).max() == 64
    assert q[1:].min() >= o8.TAIL_MIN and q[1:].max() <= o8.TAIL_MAX
    X = o8.digits_to_X(q)
    for i in range(P.shape[0]):
        for k in (0, 1, 5, 100, 255):
            y = Fraction(float(P[i, k])) * Fraction(float(rinv[i]))
            assert X[i, k] == round(y * 2 ** 46)                                  # round half to even, like rint
            assert abs(y - Fraction(int(X[i, k]), 2 ** 46)) <= Fraction(1, 2 ** 47)
            assert Fraction(int(X[i, k]), 2 ** 46) == sum(Fraction(int(q[s, i, k]), 2 ** (6 + 8 * s)) for s in range(6))


def test_near_bound_digits_round_trip():
    rng = np.random.default_rng(6)
    q = o8.near_bound_digits(rng, 8, 128)
    P = o8.digits_to_values(q)
    e, _, rinv = om.row_exponents(P)
    assert np.all(e == 0)
    assert np.array_equal(o8.slice_rows(P, rinv), q)


def test_non_finite_entries_give_zero_digits():
    P = np.ones((3, 64))
    P[0, 3], P[1, 7], P[2, 9] = np.nan, np.inf, -np.inf
    _, rscale, rinv = om.row_exponents(P)
    assert np.all(np.isnan(rscale))
    assert not o8.slice_rows(P, rinv).any()


def test_integer_ranges():
    """what the kernel needs of its integers, at the largest K it accepts: the int32 diagonals, the 2^51 range of the
    exact int64 -> fp64 conversion (in fact |h|, |l| < 2^47), and why the int32 pair pre-combination is not used"""
    K = o8.MAX_K
    assert [o8.acc_bound(d, K) for d in range(6)] == [K * b for b in (4096, 16384, 32768, 49152, 65536, 81920)]
    assert max(o8.acc_bound(d, K) for d in range(6)) < 2 ** 31
    assert max(o8.acc_bound(d, 2 * K) for d in range(6)) >= 2 ** 31             # the bound fails at the next power of two
    h, l = o8.word_bounds(K)
    assert h < 2 ** 47 and l < 2 ** 47
    assert 256 * o8.acc_bound(1, 512) >= 2 ** 31                                 # 256 ACC overflows int32 from K = 512


def test_near_bound_accumulators_at_the_largest_k():
    """aligned near-maximal digits at K = 16384: the model's accumulators and words stay in range (asserted inside)"""
    rng = np.random.default_rng(7)
    q = o8.near_bound_digits(rng, 3, o8.MAX_K)
    acc = o8.accumulators(q, q)
    assert np.abs(acc[5]).max() > 2 ** 30
    h, l = o8.words(acc)
    assert np.abs(h).max() < 2 ** 47 and np.abs(l).max() < 2 ** 47


def test_term_bound():
    """about 2^-43.4: 6x looser than seven 7-bit slices, 18x tighter than six 7-bit slices"""
    b = o8.term_bound()
    assert abs(math.log2(b) - (-43.4)) < 0.02
    assert b < om.trunc_bound(6, 0, 0, 1) / 16 and b < om.trunc_bound(7, 0, 0, 1) * 7


@pytest.mark.parametrize("K", KS)
def test_model_is_within_the_exact_bound(K):
    rng = np.random.default_rng(K)
    m, n = (6, 5) if K >= 4096 else (12, 9)
    A, B = _operands(rng, m, K), _operands(rng, n, K)
    C0 = rng.standard_normal((m, n)) * np.ldexp(1.0, rng.integers(-20, 40, (m, n)))
    sign = -1.0 if K % 3 else 1.0
    got = _model(A, B, C0, sign)
    ea, eb = om.row_exponents(A)[0], om.row_exponents(B)[0]
    for i in range(m):
        for j in range(n):
            ex = om.exact_entry(C0[i, j], A[i], B[j], sign)
            assert abs(Fraction(float(got[i, j])) - ex) <= o8.result_bound(ea[i], eb[j], K, got[i, j]), (i, j)


def test_formats_agree_within_their_bounds():
    """the eight-bit and the seven-slice seven-bit models of one product differ by less than the sum of their bounds"""
    rng = np.random.default_rng(9)
    K = 512
    A, B = _operands(rng, 10, K, -3, 3), _operands(rng, 7, K, -3, 3)
    C0 = np.zeros((10, 7))
    got8 = _model(A, B, C0, 1.0)
    ws = om.Workspace(7, K, 128 + 7).put(A).put(B, 128)
    flat = om.expected_update(ws, C0.T.reshape(-1), 10, 10, 7, 1.0, 0, om.column_rows(7, 32, 128), np.ones((10, 7), bool),
                              True, False)
    got7 = flat.reshape(7, 10).T
    ea, eb = om.row_exponents(A)[0], om.row_exponents(B)[0]
    sc = np.ldexp(1.0, ea[:, None] + eb[None, :]) * K
    assert np.all(np.abs(got8 - got7) <= sc * (float(o8.term_bound()) + float(om.trunc_bound(7, 0, 0, 1)) + 2.0 ** -51))
