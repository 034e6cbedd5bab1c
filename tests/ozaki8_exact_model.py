"""Exact model of the eight-bit format of the int8-slice update (``ozaki8_update_kernel``, the BITS = 8 branch of
ozaki_slice_kernel and oz_combine in abstractgps.jl_b200/csrc/umma_ozaki.cu).

The row exponents, the tile walks and the fma of the drain are those of the seven-bit format (tests/ozaki_exact_model.py,
reused here); what differs is operation by operation:

* ``slice_rows``  -- X = rint(y 2^46) held as an int64 (|X| <= 2^46; 0 for a non-finite entry), the balanced bytes
                     q_5 .. q_1 in [-128, 127] peeled off the low end (X = (X - q) / 256, exact) and q_0 = X, |q_0| <= 64;
                     y = sum_s q_s 2^-(6+8s) to within 2^-47
* ``accumulators`` -- ACC_d = sum_{s+t=d} q_s q_t' for d < 6, 21 slice pairs, int32
* ``words``/``combine`` -- h = (ACC_0 256 + ACC_1) 256 + ACC_2, l = (ACC_3 256 + ACC_4) 256 + ACC_5 (int64),
                     v = fma(l, 2^-24, h): the one rounding before the drain
* ``scale_products`` -- the drain's p_ij = (sign 2^e_i 2^-28) 2^e_j

plus the bounds the kernel relies on (``acc_bound``, ``word_bounds``) and the truncation bound of one product term.
"""
from fractions import Fraction

import numpy as np

import ozaki_exact_model as om

S = 6
BITS = 8
MAX_K = 16384                    # OZ8_MAX_K: the int32 accumulators are exact up to this K
LO_SCALE = 2.0 ** -24
SCALE = 1.0 / 268435456.0        # 2^-28 = 2^-12 (two leading digit weights) * 2^-16 (v = 2^16 sum_d ACC_d 256^-d)
Q0_MAX, TAIL_MIN, TAIL_MAX = 64, -128, 127


def acc_bound(d, K):
    """|ACC_d| <= K sum_{s+t=d} |q_s|max |q_t|max with |q_0| <= 64 and |q_s>0| <= 128; d = 5 gives 5 2^14 K"""
    mag = lambda s: Q0_MAX if s == 0 else 128
    return K * sum(mag(s) * mag(d - s) for s in range(S) if 0 <= d - s < S)


def word_bounds(K):
    """bounds of |h| and |l| from acc_bound"""
    b = [acc_bound(d, K) for d in range(S)]
    return b[0] * 65536 + b[1] * 256 + b[2], b[3] * 65536 + b[4] * 256 + b[5]


# ---- pre-pass ---------------------------------------------------------------------------------------------------------
def slice_rows(P, rinv):
    """ozaki_slice_kernel<6, 8>: q[6, m, K] (int64).  y = x * rinv is the kernel's own multiply (exact but for subnormal
    underflow); y 2^46 is exact; rint rounds half to even like __double2ll_rn."""
    P = np.asarray(P, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        t = (P * rinv[:, None]) * 2.0 ** 46
        ok = np.abs(t) <= 2.0 ** 46
        X = np.where(ok, np.rint(np.where(ok, t, 0.0)), 0.0).astype(np.int64)
    q = np.empty((S,) + P.shape, dtype=np.int64)
    for s in range(S - 1, 0, -1):
        q[s] = ((X & 0xFF) ^ 0x80) - 0x80            # the low byte, sign-extended
        X = (X - q[s]) >> 8                           # exact: X - q is a multiple of 256
    q[0] = X
    return q


def digits_to_X(q):
    X = np.zeros(q.shape[1:], dtype=np.int64)
    for s in range(S):
        X = X * 256 + q[s]
    return X


def digits_to_values(q):
    """the operand values whose digits are exactly q: x = X 2^-46 (X < 2^47, so x is an fp64 number)"""
    X = digits_to_X(q)
    assert np.abs(X).max(initial=0) <= 2 ** 46
    return np.ldexp(X.astype(np.float64), -46)


def near_bound_digits(rng, m, K, lead=(56, 63), tail=(120, 127)):
    """digits with one sign per row, |q_0| in lead, |q_s>0| in tail: the accumulators reach about 61 % of the int32
    range at K = 16384 and every row maximum lies in [0.5, 1), so its row exponent is 0 and the slicer reproduces q"""
    sgn = np.where(rng.random((m, 1)) < 0.5, -1, 1)
    q = np.empty((S, m, K), dtype=np.int64)
    q[0] = rng.integers(lead[0], lead[1] + 1, (m, K)) * sgn
    q[1:] = rng.integers(tail[0], tail[1] + 1, (S - 1, m, K)) * sgn[None]
    return q


# ---- integer part -----------------------------------------------------------------------------------------------------
def accumulators(qa, qb):
    """ACC_d for d < 6.  The float64 matmuls are exact: every partial sum is an integer below K 2^14 < 2^53."""
    K = qa.shape[2]
    assert K * 128 * 128 < 2 ** 53
    fa, fb = qa.astype(np.float64), qb.astype(np.float64)
    acc = np.zeros((S, qa.shape[1], qb.shape[1]), dtype=np.int64)
    for s in range(S):
        for t in range(S - s):
            acc[s + t] += (fa[s] @ fb[t].T).astype(np.int64)
    assert np.abs(acc).max(initial=0) < 2 ** 31, "an int32 accumulator would wrap"
    return acc


def words(acc):
    a = acc.astype(np.int64)
    return (a[0] * 256 + a[1]) * 256 + a[2], (a[3] * 256 + a[4]) * 256 + a[5]


def combine(acc):
    """v = fma(f64(l), 2^-24, f64(h)): both conversions exact (|h|, |l| < 2^51, asserted), l 2^-24 exact, one rounding"""
    h, l = words(acc)
    assert np.abs(h).max(initial=0) < 2 ** 51 and np.abs(l).max(initial=0) < 2 ** 51
    return l.astype(np.float64) * LO_SCALE + h.astype(np.float64)


def scale_products(sign, rs_a, rs_b):
    with np.errstate(invalid="ignore", over="ignore", under="ignore"):
        return (sign * rs_a * SCALE)[:, None] * rs_b[None, :]


# ---- the whole launch -------------------------------------------------------------------------------------------------
class Workspace(om.Workspace):
    def __init__(self, K, rows):
        super().__init__(S, K, rows)

    def put(self, P, row0=0):
        P = np.asarray(P, dtype=np.float64)
        _, rscale, rinv = om.row_exponents(P)
        self.q[:, row0:row0 + P.shape[0]] = slice_rows(P, rinv)
        self.rscale[row0:row0 + P.shape[0]] = rscale
        return self


def expected_update(ws, C_store, ldc, M, N, sign, a_off, col_rows, owned, base=0):
    """C_store: the 1-d buffer the kernel sees (column-major C at element `base`); returns a copy in which exactly the
    owned entries of the M x N block hold the kernel's result"""
    out = np.array(C_store, copy=True)
    for c0 in range(0, N, 256):
        cols = np.arange(c0, min(N, c0 + 256))
        own = owned[:, cols]
        rsel = np.nonzero(own.any(1))[0]
        if rsel.size == 0:
            continue
        rows = rsel + a_off
        v = combine(accumulators(ws.q[:, rows], ws.q[:, col_rows[cols]]))
        p = scale_products(sign, ws.rscale[rows], ws.rscale[col_rows[cols]])
        idx = base + rsel[:, None] + cols[None, :] * ldc
        new = om.drain(v, p, out[idx], False)
        own = own[rsel]
        out[idx[own]] = new[own]
    return out


# ---- bounds ---------------------------------------------------------------------------------------------------------------
def term_bound():
    """|a b - (sum of the computed diagonals)| for |a|, |b| < 1: the two representation errors (|a - a~| <= 2^-47,
    |a~| <= 1 + 2^-47) and the dropped diagonals d = 6 .. 10, each at most (number of tail pairs) 2^14 2^-(12+8d)"""
    rep = Fraction(1, 2 ** 47) * (2 + Fraction(1, 2 ** 47))
    dropped = sum(Fraction(n * 2 ** 14, 2 ** (12 + 8 * d)) for d, n in zip(range(6, 11), (5, 4, 3, 2, 1)))
    return rep + dropped


def result_bound(e_i, e_j, K, result):
    """term_bound K 2^(e_i+e_j) plus the rounding of v (relative 2^-53 of at most 2^(e_i+e_j) K (1 + 2^-46)) and of the
    fma (half an ulp of the result); below 2^-1074 the drain's scale 2^(e_i+e_j-28) flushes and the product is lost"""
    sc = Fraction(2) ** (int(e_i) + int(e_j)) * K
    b = term_bound() * sc + sc * Fraction(1, 2 ** 52) + Fraction(float(np.spacing(abs(float(result))))) / 2
    if int(e_i) + int(e_j) - 28 < -1074:
        b += sc * Fraction(101, 100)
    return b
