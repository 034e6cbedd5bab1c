"""CPU model of the arithmetic of the int8-slice SYRK (abstractgps.jl_b200/csrc/umma_ozaki.cu): row-exponent
scaling, error-free 7-bit slicing (ozaki_slice_kernel), exact int32 accumulation per diagonal d = s + t (what the
stacked-B MMAs leave in the accumulators), and the two fp64 recombinations of the epilogue -- plain Horner (AGP_OZAKI_EPI=0) and the
int32 pair pre-combination that is the default for S = 7, K <= 512 (AGP_OZAKI_EPI=1).  Checks the bounds the kernel relies
on: slices stay in [-64, 64], accumulators and pairs fit int32 for K <= 512 (and the pair does NOT fit at K = 1024, which is
why the host falls back), both recombinations agree with exact integer arithmetic to fp64 rounding, and the final update
meets the 2^-7S truncation bound."""
from fractions import Fraction

import numpy as np
import pytest


def slice_rows(P, S):
    """ozaki_rowscale_kernel + ozaki_slice_kernel: returns (q[S, m, K] int64, scale[m])."""
    mx = np.abs(P).max(1)
    e = np.where(mx > 0, np.frexp(mx)[1], 0)
    scale = np.ldexp(1.0, e)
    r = P / scale[:, None]
    q = np.empty((S,) + P.shape, dtype=np.int64)
    up = 64.0
    for s in range(S):
        qs = np.rint(r * up)
        r = r - qs / up          # exact in fp64 (fma(-q, dn, r) in the kernel)
        q[s] = qs.astype(np.int64)
        up *= 128.0
    return q, scale, r


def accumulators(qa, qb, S):
    """ACC_d[i, j] = sum_{s + t = d} sum_k qa[s, i, k] qb[t, j, k], d = 0 .. S-1 (only s + t <= S-1 is computed)."""
    acc = np.zeros((S, qa.shape[1], qb.shape[1]), dtype=np.int64)
    for s in range(S):
        for t in range(S - s):
            acc[s + t] += qa[s] @ qb[t].T
    return acc


def horner_plain(acc):
    S = acc.shape[0]
    v = acc[S - 1].astype(np.float64)
    for d in range(S - 2, -1, -1):
        v = v * (1.0 / 128.0) + acc[d].astype(np.float64)  # fma in the kernel; the product by 2^-7 is exact
    return v


def horner_pairs(acc):
    """the default epilogue: t_j = 128 ACC_2j + ACC_2j+1 in int32, then Horner over the pairs (+ the odd term)."""
    S = acc.shape[0]
    a32 = acc.astype(np.int32)
    pair = lambda d: (a32[d] * np.int32(128) + a32[d + 1])  # int32 arithmetic, wraps like the device would
    if S & 1:
        v = a32[S - 1].astype(np.float64)
        v = v * (1.0 / 128.0) + pair(S - 3).astype(np.float64)
        for d in range(S - 5, -1, -2):
            v = v * (1.0 / 16384.0) + pair(d).astype(np.float64)
    else:
        v = pair(S - 2).astype(np.float64)
        for d in range(S - 4, -1, -2):
            v = v * (1.0 / 16384.0) + pair(d).astype(np.float64)
    return v * (1.0 / 128.0)


def exact_value(acc, i, j):
    S = acc.shape[0]
    return sum(Fraction(int(acc[d, i, j]), 128 ** d) for d in range(S))


@pytest.mark.parametrize("S", [5, 6, 7, 8])
def test_slices_accumulators_and_both_epilogues(S):
    rng = np.random.default_rng(S)
    m, K = 48, 512
    P = rng.standard_normal((m, K)) * np.exp(rng.uniform(-6, 6, (m, 1)))
    q, scale, resid = slice_rows(P, S)
    assert np.abs(q).max() <= 64
    assert np.abs(resid).max() <= 2.0 ** (-7 * S)  # what the S slices leave behind, relative to the row scale
    acc = accumulators(q, q, S)
    for d in range(S):
        assert np.abs(acc[d]).max() <= (d + 1) * K * 64 * 64 < 2 ** 31
    v0, v1 = horner_plain(acc), horner_pairs(acc)
    for (i, j) in [(0, 0), (3, 17), (47, 1), (20, 20), (5, 44)]:
        ex = exact_value(acc, i, j)
        for v in (v0, v1):
            assert abs(Fraction(float(v[i, j])) - ex) <= abs(ex) * Fraction(1, 2 ** 51) + Fraction(1, 2 ** 60)
    # the update itself: scale_i scale_j / 4096 * v  vs  fp64 P P'
    got = v1 * (scale[:, None] / 4096.0) * scale[None, :]
    want = P @ P.T
    bound = (2.0 ** (-7 * S + 3)) * np.outer(scale, scale) * K + 4e-16 * np.abs(want) + 1e-300
    assert np.all(np.abs(got - want) <= bound)


@pytest.mark.parametrize("S", [5, 6, 7, 8])
def test_pair_bound_holds_at_k512_and_fails_at_k1024(S):
    """worst case: every slice entry +-64 with aligned signs.  K = 512: every pair fits int32 (exact result);
    K = 1024: the pair of diagonals (4, 5) wraps for S >= 6 -- the launcher must not use the pair epilogue there."""
    for K, must_fit in ((512, True), (1024, False)):
        q = np.full((S, 2, K), 64, dtype=np.int64)
        acc = accumulators(q, q, S)
        assert np.abs(acc).max() < 2 ** 31  # the accumulators themselves always fit
        v0, v1 = horner_plain(acc), horner_pairs(acc)
        fits = np.array_equal(v0, v1) or np.allclose(v0, v1, rtol=1e-15, atol=0)
        if must_fit:
            assert fits
        elif S >= 6:
            assert not fits


def test_umma_noswizzle_chunk_layout_halves():
    """ozaki_slice_kernel's bulk layout: byte offset of (row, k) inside a 4096-byte chunk; the cluster variant multicasts
    bytes [0, 2048) from CTA 0 and [2048, 4096) from CTA 1 and relies on these being rows 0-63 and 64-127."""
    def off(row, kbyte):
        g, r8, h = (row & 127) >> 3, row & 7, (kbyte >> 4) & 1
        return ((g * 2 + h) * 8 + r8) * 16 + (kbyte & 15)
    seen = set()
    for row in range(128):
        for kb in range(32):
            o = off(row, kb)
            assert (o < 2048) == (row < 64)
            seen.add(o)
    assert seen == set(range(4096))


# ---- the drain: exact int64 words + magic-number conversion + ONE rounding --------------------------------
MAGIC = 0x4338000000000000        # bit pattern of 2^52 + 2^51
MAGIC_D = 6755399441055744.0      # 2^52 + 2^51


def i64_to_f64_exact(x):
    """the device's i64_to_f64_exact: as_double(x + MAGIC) - (2^52 + 2^51), exact for |x| < 2^51"""
    bits = (np.asarray(x, dtype=np.int64) + np.int64(MAGIC)).astype(np.int64)
    return bits.view(np.float64) - MAGIC_D


def oz_combine(acc, pair32):
    """oz_combine<S, BN, PAIR32> of csrc/umma_ozaki.cu on a [S, ...] int64 array of accumulators: value = sum_d acc_d 128^(3-d)"""
    S = acc.shape[0]
    a = acc.astype(np.int64)
    if S <= 4:
        h = a[0].copy()
        for d in range(1, S):
            h = h * 128 + a[d]
        for _ in range(S, 4):
            h = h * 128
        return i64_to_f64_exact(h)
    if pair32:
        a32 = acc.astype(np.int32)
        t = lambda d: (a32[d] * np.int32(128) + a32[d + 1]).astype(np.int64)   # int32 arithmetic, wraps like the device
        h = t(0) * 16384 + t(2)
        if S == 5:
            l = a[4]
        elif S == 6:
            l = t(4)
        elif S == 7:
            l = t(4) * 128 + a[6]
        else:
            l = t(4) * 16384 + t(6)
    else:
        h = ((a[0] * 128 + a[1]) * 128 + a[2]) * 128 + a[3]
        l = a[4].copy()
        for d in range(5, S):
            l = l * 128 + a[d]
    lo_scale = {5: 1.0 / 128, 6: 1.0 / 16384, 7: 1.0 / 2097152, 8: 1.0 / 268435456}[S]
    hh, ll = i64_to_f64_exact(h), i64_to_f64_exact(l)
    # fma(ll, lo_scale, hh): ll * lo_scale is exact (power of two), so the fma equals one correctly rounded addition
    return (ll * lo_scale) + hh


def test_magic_number_conversion_is_exact_below_2_pow_51():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.integers(-(2 ** 51) + 1, 2 ** 51 - 1, 10000), [0, 1, -1, 2 ** 51 - 1, -(2 ** 51) + 1, 2 ** 45 + 3]])
    assert np.array_equal(i64_to_f64_exact(x), x.astype(np.float64))          # |x| < 2^53: the cast is exact too
    assert all(Fraction(float(v)) == int(u) for u, v in zip(x[:200], i64_to_f64_exact(x[:200])))


@pytest.mark.parametrize("S", [3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("K,pair32", [(512, True), (512, False), (4096, False), (32768, False)])
def test_v3_drain_is_exact_up_to_one_rounding(S, K, pair32):
    """worst-case-magnitude and random accumulators: the int64 words stay below 2^51 for K <= 32768 (the bound
    ozaki_update_ex enforces), both integer paths agree, and the result equals the exact rational value rounded once"""
    rng = np.random.default_rng(S * 100 + K % 97)
    lim = np.array([(d + 1) * K * 4096 for d in range(S)], dtype=np.int64)
    assert lim.max() < 2 ** 31
    acc = np.stack([rng.integers(-lim[d], lim[d] + 1, 64) for d in range(S)])
    acc[:, 0] = lim           # all accumulators at their positive bound
    acc[:, 1] = -lim
    # word bounds
    a = acc.astype(object)
    h = sum(a[d] * 128 ** (3 - d) for d in range(min(S, 4)))
    assert max(abs(int(v)) for v in h) < 2 ** 51
    if S > 4:
        l = sum(a[d] * 128 ** (S - 1 - d) for d in range(4, S))
        assert max(abs(int(v)) for v in l) < 2 ** 51
    got = oz_combine(acc, pair32 and K <= 512)
    for j in range(acc.shape[1]):
        ex = sum(Fraction(int(acc[d, j]), 1) * Fraction(128) ** (3 - d) for d in range(S))
        g = Fraction(float(got[j]))
        assert abs(g - ex) <= abs(ex) * Fraction(1, 2 ** 53) + Fraction(1, 2 ** 80), (S, K, j)
    if S > 4 and K <= 512:
        assert np.array_equal(oz_combine(acc, True), oz_combine(acc, False))   # the pair form is exact for K <= 512


@pytest.mark.parametrize("S,bits", [(3, 21), (4, 28)])
def test_fp32_operands_are_covered_by_short_splits(S, bits):
    """fp32 panels sliced into S 7-bit digits: 4 slices (28 bits) hold the 24-bit significand of every element with |x| >= 2^-4 of
    the row scale exactly; the product with the d <= S-1 diagonals reproduces fp32-precision results"""
    rng = np.random.default_rng(S)
    m, K = 32, 512
    P = (rng.standard_normal((m, K)) * np.exp(rng.uniform(-3, 3, (m, 1)))).astype(np.float32).astype(np.float64)
    q, scale, resid = slice_rows(P, S)
    assert np.abs(q).max() <= 64
    assert np.abs(resid).max() <= 2.0 ** (-7 * S)
    if S == 4:   # 4 slices resolve 2^-27 of the row scale 2^e: a 24-bit significand with |x| >= 2^(e-4) is held exactly
        big = np.abs(P) >= scale[:, None] * 2.0 ** -4
        assert np.all(resid[big] == 0.0)
    acc = accumulators(q, q, S)
    v = oz_combine(acc, False)                      # value * 128^3
    got = v * (scale[:, None] * 2.0 ** -33) * scale[None, :]
    want = P @ P.T
    bound = (2.0 ** (-7 * S + 3)) * np.outer(scale, scale) * K + 1e-300
    assert np.all(np.abs(got - want) <= bound)
    assert np.all(np.abs(got - want) <= 2.0 ** (-bits + 6) * np.outer(scale, scale) * np.sqrt(K) * 8 + 1e-300)


def test_v3_slice_layout_matches_the_producer_addressing():
    """ozaki_slice_kernel (bulk == 2) writes byte (row, k, slice s) of the panel at
         chunk = ((row >> 7) * (K >> 5) + (k >> 5)) * S + s,   offset = chunk * 4096 + core-matrix offset(row & 127, k & 31);
    the producer fetches, for a 128-row tile at `arow` and k block kb, ONE run of S * 4096 bytes (A slices 0..S-1 in
    order) and for a BN-row strip at `brow` (BN = 64 or 32) S pieces of BN * 32 bytes at stride 4096 -- both must see
    exactly their rows."""
    S, K, rows = 7, 128, 512
    nkb = K >> 5

    def core(row, kbyte):
        g, r8, h = (row & 127) >> 3, row & 7, (kbyte >> 4) & 1
        return ((g * 2 + h) * 8 + r8) * 16 + (kbyte & 15)

    buf = np.full(((rows >> 7) * nkb * S * 4096, 3), -1, dtype=np.int64)   # (row, k, slice) stored at every byte
    for row in range(rows):
        for k in range(K):
            for s in range(S):
                chunk = ((row >> 7) * nkb + (k >> 5)) * S + s
                buf[chunk * 4096 + core(row, k & 31)] = (row, k, s)
    assert (buf[:, 0] >= 0).all()                                        # every byte written exactly once (a bijection)
    rb_bytes = nkb * S * 4096
    for arow, kb in ((0, 0), (128, 3), (384, 1)):
        a = buf[(arow >> 7) * rb_bytes + kb * S * 4096:][: S * 4096]
        for sl in range(S):
            tile = a[sl * 4096:(sl + 1) * 4096]
            assert set(tile[:, 2]) == {sl} and set(tile[:, 0]) == set(range(arow, arow + 128))
            assert set(tile[:, 1]) == set(range(kb * 32, kb * 32 + 32))
            # inside the tile: the no-swizzle K-major core-matrix layout of the MMA descriptors (SBO 256 B, LBO 128 B)
            r, k = 77, kb * 32 + 21
            assert tuple(tile[core(r, 21)]) == (arow + r, k, sl)
    for BN, brow, kb in ((64, 0, 2), (64, 64, 0), (64, 192, 3), (64, 448, 1), (32, 32, 1), (32, 96, 2), (32, 416, 0)):
        base = (brow >> 7) * rb_bytes + (brow & 127) * 32 + kb * S * 4096
        for sl in range(S):
            piece = buf[base + sl * 4096:][:BN * 32]
            assert set(piece[:, 2]) == {sl} and set(piece[:, 0]) == set(range(brow, brow + BN))
            assert set(piece[:, 1]) == set(range(kb * 32, kb * 32 + 32))
