"""Exact model of the int8-slice update ``ozaki_syrk_wgmma_kernel`` (abstractgps.jl_b200/csrc/umma_ozaki.cu).

Every step of the kernel before its epilogue is exact: the row exponent, the 7-bit slicing, the int32 MMA accumulators and
the int64 recombination.  The only roundings are the conversion of the two int64 words to one fp64 value and the fma of the
drain (plus the fp32 store for fp32 C).  So the kernel's output is predictable bit for bit, and this module predicts it,
operation by operation:

* ``row_exponents``   -- ozaki_rowscale_kernel: 2^e per operand row (|x| < 2^e), e >= -1022; NaN for a row with a NaN or
                         +-Inf entry or a maximum >= 2^1023
* ``slice_rows``      -- ozaki_slice_kernel: x 2^-e = sum_s q_s 2^-(6+7s), q_s in [-64, 64]; non-finite entries give 0 digits
* ``accumulators``    -- ACC_d = sum_{s+t=d} q_s q_t' for d < S (what the S(S+1)/2 MMAs leave in the int32 registers)
* ``combine``         -- oz_combine: the words h (d < 4) and l (d >= 4), the int32 pair form, one fp64 rounding
* ``drain``           -- oz_drain: fma(v, (sign 2^e_i 2^-33) 2^e_j, C_old), rounded to fp32 for fp32 C
* ``owned_*``, ``column_rows`` -- which output tiles each walk writes, and the panel row of every column
* ``expected_update`` -- all of the above on a column-major C buffer; everything the kernel must not write is copied

plus exact rational references (``exact_entry``) and the truncation bound (``trunc_bound``) the CPU tests hold the model to.
"""
from fractions import Fraction

import numpy as np

BM = 128                         # rows per output tile
LO_SCALE = {5: 2.0 ** -7, 6: 2.0 ** -14, 7: 2.0 ** -21, 8: 2.0 ** -28}


def tile_width(S):
    """BN: the accumulators of S blocks of 64 x BN int32 must fit the registers"""
    return 64 if S <= 4 else 32


def pair32_used(S, K, epi_env=None):
    """the launcher's drain choice: int32 pair pre-combination for S >= 5, K <= 512 unless AGP_OZAKI_EPI=0"""
    return S >= 5 and K <= 512 and not (epi_env is not None and int(epi_env) == 0)


def ceil128(n):
    return (n + BM - 1) // BM * BM


# ---- pre-passes -------------------------------------------------------------------------------------------------------
def row_exponents(P):
    """ozaki_rowscale_kernel on the rows of P (float64 values; fp32 operands converted exactly).
    Returns (e, rscale, rinv): rscale = 2^e with |x| < 2^e for every entry of the row, e clamped to >= -1022 so that
    rinv = 2^-e stays finite (scaling a subnormal row by it is exact); a row holding a NaN or +-Inf, or whose maximum is
    >= 2^1023 (2^e would overflow), gets rscale = NaN and rinv = 0, so every output it touches is NaN."""
    P = np.asarray(P, dtype=np.float64)
    a = np.abs(P)
    a = np.where(np.isnan(a), np.inf, a)               # the kernel maps NaN to +inf before its fmax reduction
    mx = a.max(1) if P.shape[1] else np.zeros(P.shape[0])
    ok = (mx > 0) & np.isfinite(mx)
    e = np.where(ok, np.frexp(np.where(ok, mx, 1.0))[1], 0).astype(np.int64)
    e = np.maximum(e, -1022)
    bad = ~(mx < 2.0 ** 1023)
    ec = np.where(bad, 0, e)
    rscale = np.where(bad, np.nan, np.ldexp(1.0, ec))
    rinv = np.where(bad, 0.0, np.ldexp(1.0, -ec))
    return ec, rscale, rinv


def slice_rows(P, S, rinv):
    """ozaki_slice_kernel: q[S, m, K] (int64) and the residual r[m, K] left after S digits, both relative to the row
    scale.  r = x * rinv is exact but for subnormal underflow (the kernel's own multiply, reproduced here); each digit is
    q = rint(r 2^(6+7s)), r -= q 2^-(6+7s) (the kernel's fma: q 2^-(6+7s) is exact, so one rounding, and that one is exact
    too).  A digit outside [-64, 64] -- only a NaN or +-Inf entry can produce one -- is stored as 0."""
    P = np.asarray(P, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        r = P * rinv[:, None]
        q = np.empty((S,) + P.shape, dtype=np.int64)
        up, dn = 64.0, 1.0 / 64.0
        for s in range(S):
            qs = np.rint(r * up)
            qs = np.where(np.abs(qs) <= 64.0, qs, 0.0)
            r = r - qs * dn
            q[s] = qs.astype(np.int64)
            up *= 128.0
            dn *= 1.0 / 128.0
    return q, r


def digits_to_values(q):
    """the operand values whose S digits are exactly q[S, m, K]: x = sum_s q_s 2^-(6+7s).  Asserts that x is an fp64
    number (the digit string fits the 53-bit significand), so the slicer can return q unchanged."""
    S = q.shape[0]
    X = np.zeros(q.shape[1:], dtype=np.int64)
    for s in range(S):
        X = X * 128 + q[s]
    F = X.astype(np.float64)
    assert np.array_equal(F.astype(np.int64), X), "digit string longer than an fp64 significand"
    return np.ldexp(F, -(6 + 7 * (S - 1)))


def near_bound_digits(rng, S, m, K, lo=60, hi=63):
    """digits with lo <= |q| <= hi, one sign per row (aligned over slices and k): the accumulators reach
    (d+1) K hi^2 and the int64 words approach their bounds.  hi < 64 keeps every remainder below half a digit, so the
    slicer reproduces them; for S = 8 the last digit is a multiple of 4 so that the value fits 53 bits."""
    sgn = np.where(rng.random((m, 1)) < 0.5, -1, 1)
    q = rng.integers(lo, hi + 1, (S, m, K)) * sgn[None]
    if S == 8:
        q[S - 1] = (np.abs(q[S - 1]) // 4 * 4) * sgn
        assert np.all(np.abs(q[S - 1]) >= lo)
    return q


# ---- integer part -----------------------------------------------------------------------------------------------------
def accumulators(qa, qb):
    """ACC_d[i, j] = sum_{s+t=d} sum_k qa[s, i, k] qb[t, j, k] for d < S (the diagonals the kernel computes).  The float64
    matmuls are exact: every product and partial sum is an integer of magnitude <= K 64^2 < 2^53."""
    S, K = qa.shape[0], qa.shape[2]
    assert K * 64 * 64 < 2 ** 53
    fa, fb = qa.astype(np.float64), qb.astype(np.float64)
    acc = np.zeros((S, qa.shape[1], qb.shape[1]), dtype=np.int64)
    for s in range(S):
        for t in range(S - s):
            acc[s + t] += (fa[s] @ fb[t].T).astype(np.int64)
    assert np.abs(acc).max(initial=0) < 2 ** 31, "an int32 accumulator would wrap"
    return acc


def words(acc, pair32):
    """(h, l) int64 as oz_combine forms them.  S <= 4: h = sum_d ACC_d 128^(3-d), l = 0.  S >= 5: h = sum_{d<4} ACC_d
    128^(3-d), l = sum_{d>=4} ACC_d 128^(S-1-d); pair32 forms 128 ACC_d + ACC_d+1 in int32 first (wrapping like the
    device, which is harmless only for K <= 512)."""
    S = acc.shape[0]
    a = acc.astype(np.int64)
    if S <= 4:
        h = a[0].copy()
        for d in range(1, S):
            h = h * 128 + a[d]
        for _ in range(S, 4):
            h = h * 128
        return h, np.zeros_like(h)
    if pair32:
        a32 = acc.astype(np.int32)
        t = lambda d: (a32[d] * np.int32(128) + a32[d + 1]).astype(np.int64)
        h = t(0) * 16384 + t(2)
        l = {5: lambda: a[4], 6: lambda: t(4), 7: lambda: t(4) * 128 + a[6], 8: lambda: t(4) * 16384 + t(6)}[S]()
        return h, l
    h = ((a[0] * 128 + a[1]) * 128 + a[2]) * 128 + a[3]
    l = a[4].copy()
    for d in range(5, S):
        l = l * 128 + a[d]
    return h, l


def combine(acc, pair32):
    """oz_combine: v = fma(f64(l), LO_SCALE, f64(h)), the value sum_d ACC_d 128^(3-d) rounded once.  The int64 -> fp64
    conversion of the kernel is exact below 2^51, which is asserted; l * LO_SCALE is exact, so numpy's multiply-add
    rounds exactly once, like the fma."""
    S = acc.shape[0]
    h, l = words(acc, pair32)
    assert np.abs(h).max(initial=0) < 2 ** 51 and np.abs(l).max(initial=0) < 2 ** 51
    if S <= 4:
        return h.astype(np.float64)
    return l.astype(np.float64) * LO_SCALE[S] + h.astype(np.float64)


def exact_fma(x, y, z):
    """fma(x, y, z) in fp64 with one rounding, through exact rationals (CPython's int / int division rounds correctly)"""
    if not (np.isfinite(x) and np.isfinite(y) and np.isfinite(z)):
        return float(np.float64(x) * np.float64(y) + np.float64(z))
    ex = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
    return float(ex) if ex != 0 else float(np.float64(x) * np.float64(y) + np.float64(z))


def drain(v, p, c_old, c_is_float):
    """C_new = fma(v, p, C_old), stored as fp32 for fp32 C.  v p is exact wherever it is a normal number (p is a power of
    two), so multiply-then-add is the fma there; products that land in the subnormal range go through ``exact_fma``."""
    c64 = np.asarray(c_old, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore", under="ignore"):
        prod = v * p
        out = prod + c64
        tiny = np.isfinite(prod) & (prod != 0) & (np.abs(prod) < 2.0 ** -1022)
    for idx in zip(*np.nonzero(tiny)):
        out[idx] = exact_fma(v[idx], p[idx], c64[idx])
    return out.astype(np.float32) if c_is_float else out


def scale_products(sign, rs_a, rs_b):
    """the drain's p_ij = (sign * 2^e_i * 2^-33) * 2^e_j, evaluated in the kernel's order"""
    with np.errstate(invalid="ignore", over="ignore", under="ignore"):
        return (sign * rs_a * (1.0 / 8589934592.0))[:, None] * rs_b[None, :]


# ---- tile walks ---------------------------------------------------------------------------------------------------------
def owned_lower(M, N, BN):
    """closed-form lower walk (a_off == b_off, identity column map): tile (bi, bj) is written iff bj BN < 128 (bi + 1)"""
    i, j = np.indices((M, N))
    return (j // BN) * BN < BM * (i // BM + 1)


def column_rows(N, BN, b_off, stride=0, bw=0):
    """panel row of every column n: the kernel maps strip j's first column n0 to (n0 / bw) stride + n0 % bw + b_off
    (stride 0: n0 + b_off) and the strip's columns to the consecutive rows after it"""
    bw = bw or BM
    n = np.arange(N)
    n0 = n // BN * BN
    brow = ((n0 // bw) * stride + n0 % bw if stride else n0) + b_off
    return brow + (n - n0)


def owned_table(M, N, BN, b_off, a_off, stride=0, bw=0, full=False):
    """strip-table walk: strip j owns row tiles bi >= bimin[j], the first row tile whose panel rows reach the strip's
    first column (every row tile for a rectangular product)"""
    nbi = (M + BM - 1) // BM
    i, j = np.indices((M, N))
    if full:
        return np.ones((M, N), dtype=bool)
    src0 = column_rows(N, BN, b_off, stride, bw)[(np.arange(N) // BN) * BN]
    bimin = np.where(src0 - a_off >= 0, (src0 - a_off) // BM, 0)
    bimin = np.minimum(bimin, nbi)
    return (i // BM) >= bimin[j]


# ---- the whole launch -------------------------------------------------------------------------------------------------
class Workspace:
    """slices and row scales of one slice workspace: rows [0, rows) hold operand rows placed by ``put``; rows between
    operands up to the next multiple of 128 hold zero digits (their row scale is never read by an owned entry)"""

    def __init__(self, S, K, rows):
        self.S, self.K = S, K
        self.q = np.zeros((S, ceil128(rows), K), dtype=np.int64)
        self.rscale = np.full(ceil128(rows), np.nan)

    def put(self, P, row0=0):
        P = np.asarray(P, dtype=np.float64)
        _, rscale, rinv = row_exponents(P)
        q, _ = slice_rows(P, self.S, rinv)
        self.q[:, row0:row0 + P.shape[0]] = q
        self.rscale[row0:row0 + P.shape[0]] = rscale
        return self


def expected_update(ws, C_store, ldc, M, N, sign, a_off, col_rows, owned, pair32, c_is_float, base=0):
    """C_store: the whole 1-d storage buffer the kernel sees (column-major C at element offset `base`, leading dimension
    ldc).  Returns a copy in which exactly the owned entries of the M x N block hold the kernel's result."""
    out = np.array(C_store, copy=True)
    for c0 in range(0, N, 256):  # column blocks keep the S x M x 256 accumulators small
        cols = np.arange(c0, min(N, c0 + 256))
        own = owned[:, cols]
        rsel = np.nonzero(own.any(1))[0]
        if rsel.size == 0:
            continue
        rows = rsel + a_off
        acc = accumulators(ws.q[:, rows], ws.q[:, col_rows[cols]])
        v = combine(acc, pair32)
        p = scale_products(sign, ws.rscale[rows], ws.rscale[col_rows[cols]])
        idx = base + rsel[:, None] + cols[None, :] * ldc
        new = drain(v, p, out[idx], c_is_float)
        own = own[rsel]
        out[idx[own]] = new[own]
    return out


# ---- exact references ---------------------------------------------------------------------------------------------------
def _to_ints(x):
    m, e = np.frexp(np.asarray(x, dtype=np.float64))
    return (m * 2.0 ** 53).astype(np.int64), e.astype(np.int64) - 53


def exact_dot(a, b):
    """sum_k a_k b_k of two finite float64 vectors as an exact Fraction"""
    ia, ea = _to_ints(a)
    ib, eb = _to_ints(b)
    e = ea + eb
    nz = (ia != 0) & (ib != 0)
    if not nz.any():
        return Fraction(0)
    ia, ib, e = ia[nz], ib[nz], e[nz]
    e0 = int(e.min())
    tot = sum(int(x) * int(y) << int(s) for x, y, s in zip(ia, ib, e - e0))
    return Fraction(tot) * (Fraction(2) ** e0)


def exact_entry(c_old, a_row, b_row, sign):
    """the exact rational C_old + sign * a . b"""
    return Fraction(float(c_old)) + int(sign) * exact_dot(a_row, b_row)


def trunc_bound(S, e_i, e_j, K):
    """|computed sum - exact sum| before the final roundings, for rows with |a| < 2^e_i, |b| < 2^e_j: the dropped
    diagonals d >= S contribute at most (S-1) 2^-7S (128/127) per term and the residuals of the two operands after S
    digits at most 2^-7S (1 + 2^-7S) each, so (S + 1.06) 2^-7S 2^(e_i+e_j) K"""
    return Fraction(S * 100 + 106, 100) * Fraction(2) ** (-7 * S + int(e_i) + int(e_j)) * K


def result_bound(S, e_i, e_j, K, result, c_is_float):
    """trunc_bound plus the roundings after it: v to fp64 (relative 2^-53 of at most 2^(e_i+e_j) K (1 + 2^-7S)^2), the
    fma (half an fp64 ulp of the result) and, for fp32 C, the store (half an fp32 ulp).  The drain's scale factor
    2^(e_i+e_j-33) is an fp64 number: below 2^-1074 it flushes to 0 and the whole product (< 2^(e_i+e_j) K, itself
    below 2^-1041 K) is lost."""
    sc = Fraction(2) ** (int(e_i) + int(e_j)) * K
    r = abs(float(result))
    b = trunc_bound(S, e_i, e_j, K) + sc * Fraction(1, 2 ** 52) + Fraction(float(np.spacing(r))) / 2
    if int(e_i) + int(e_j) - 33 < -1074:
        b += sc * Fraction(101, 100)
    if c_is_float:
        b += Fraction(float(np.spacing(np.float32(r)))) / 2
    return b
