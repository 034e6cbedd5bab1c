"""CPU checks of the tile-GEMM model (tests/gemm_exact_model.py): it equals a naive loop in exact rational arithmetic on
small products, its data keep every sum exact, and on the shapes the device test runs its output depends on the tile,
so a bit-exact match pins which kernel ran."""
from dataclasses import replace
from fractions import Fraction

import numpy as np
import pytest

import gemm_exact_model as gm


def _naive(g, A, B, Cbuf, tbm, tbn):
    want = Cbuf.copy()
    for m in range(g.M):
        m0 = m // tbm * tbm
        for n in range(g.N):
            n0 = n // tbn * tbn
            if g.lower_only and int(gm.col_source(g, n0)) >= m0 + tbm:
                continue
            src = int(gm.col_source(g, n))
            kend = min(g.K, m0 + tbm) if g.trmm_lower else g.K
            acc = Fraction(0)
            for k in range(kend):
                a = A[k + m * g.lda] if g.a_kmajor else A[m + k * g.lda]
                b = B[k + src * g.ldb] if g.b_kmajor else B[src + k * g.ldb]
                acc += Fraction(float(a)) * Fraction(float(b))
            c = Fraction(float(Cbuf[m + n * g.ldc])) if g.beta_one else Fraction(0)
            v = c - acc if g.alpha_neg else c + acc
            x = g.dtype(float(v))
            assert Fraction(float(x)) == v
            if v == 0:
                x = g.dtype(-0.0) if (g.dtype == np.float32 and g.alpha_neg and not g.beta_one) else g.dtype(0.0)
            want[m + n * g.ldc] = x
    return want


SMALL = [
    gm.Gemm(np.float64, 5, 7, 6, a_kmajor=1, b_kmajor=0, alpha_neg=1, beta_one=1),
    gm.Gemm(np.float64, 9, 3, 0, alpha_neg=1),
    gm.Gemm(np.float64, 11, 10, 9, lower_only=1, beta_one=1),
    gm.Gemm(np.float64, 12, 12, 12, trmm_lower=1, b_kmajor=1, alpha_neg=1),
    gm.Gemm(np.float64, 8, 6, 4, alias="A", beta_one=1),
    gm.Gemm(np.float64, 6, 9, 10, b_kmajor=1, alias="B", alpha_neg=1, beta_one=1),
    gm.Gemm(np.float64, 40, 12, 6, lower_only=1, stride=16, width=4, b_off=2, alpha_neg=1, beta_one=1),
    gm.Gemm(np.float32, 8, 5, 8, a_kmajor=1, b_kmajor=1, alpha_neg=1),
    gm.Gemm(np.float32, 12, 12, 0, alpha_neg=1),
    gm.Gemm(np.float32, 12, 7, 9, trmm_lower=1, beta_one=1),
]


@pytest.mark.parametrize("i", range(len(SMALL)))
def test_model_equals_rational_loop(i):
    """small tiles (4 x 4, 8 x 4) stand in for the kernel's, so lower_only, trmm_lower and the map all bite"""
    g = gm.with_lds(SMALL[i], extra=1)
    A, B, Cbuf = gm.make_buffers(g, np.random.default_rng(i))
    tbm, tbn = (4, 4) if i % 2 else (8, 4)
    want, own = gm.expected(g, A, B, Cbuf, tbm, tbn)
    naive = _naive(g, A, B, Cbuf, tbm, tbn)
    ut = np.uint64 if g.dtype == np.float64 else np.uint32
    assert np.array_equal(want.view(ut), naive.view(ut))


def test_fp64_cases_need_more_than_fp32_accumulation():
    """the fp64 data have partial sums above 2^24 units: an fp32 accumulator would round them"""
    g = gm.with_lds(gm.Gemm(np.float64, 64, 64, 48))
    A, B, Cbuf = gm.make_buffers(g, np.random.default_rng(0))
    a, b = gm.op_a(g, A), gm.op_b(g, B)
    prod = np.abs(a[:, :1] * b[:1, :]) / np.ldexp(1.0, (gm.low_exponent(a).min(1)[:, None] + gm.low_exponent(b).min(0)[None, :]).astype(int))
    assert prod.max() > 2.0 ** 24


def test_exactness_is_asserted():
    g = gm.with_lds(gm.Gemm(np.float32, 4, 4, 4))
    A, B, Cbuf = gm.make_buffers(g, np.random.default_rng(0))
    A = A.copy()
    A[0] = np.float32(2.0 ** 23 + 1)
    with pytest.raises(AssertionError):
        gm.expected(g, A, B, Cbuf)


@pytest.mark.parametrize("inst", gm.INSTANTIATIONS, ids=lambda t: "%s-a%d-b%d-%s" % (np.dtype(t[0]).name, t[1], t[2],
                                                                                        t[3] or "sep"))
def test_device_cases_pin_the_tile(inst):
    """on the device test's pinning products, the model under each other fp64 kernel's tile gives a different C (the
    fp32 kernels share one tile; their storage order is pinned by the NaN padding)"""
    cases = gm.pinning_cases(*inst)
    for t in gm.other_tiles(cases[0]):
        differs = False
        for i, g in enumerate(cases):
            assert gm.contract_ok(g)
            A, B, Cbuf = gm.make_buffers(g, np.random.default_rng(i))
            want, _ = gm.expected(g, A, B, Cbuf)
            other, _ = gm.expected(g, A, B, Cbuf, *t)
            differs |= not np.array_equal(want.view(np.uint64), other.view(np.uint64))
        assert differs, t


def test_device_cases_cover_the_grid():
    for inst in gm.INSTANTIATIONS:
        cases = gm.instantiation_cases(*inst)
        dt = inst[0]
        assert all(gm.contract_ok(g) for g in cases)
        Ms, Ns, Ks = {g.M for g in cases}, {g.N for g in cases}, {g.K for g in cases}
        assert Ms >= {m for m in gm.MN if dt == np.float64 or m % 4 == 0} - ({129, 300} if inst[3] == "B" else set())
        assert Ns >= {n for n in gm.MN if n > 1 or dt == np.float64} - ({129, 300} if inst[3] == "A" else set())
        assert {0, 4, 16, 48}.issubset(Ks) and max(Ks) > 1000 and any(k > 32 and k % 16 for k in Ks)
        for flag in ("lower_only", "trmm_lower", "alpha_neg", "beta_one"):
            assert {getattr(g, flag) for g in cases} == {0, 1}


def test_contract_mirror_refuses_each_clause():
    g = gm.with_lds(gm.Gemm(np.float64, 128, 128, 64, a_kmajor=1))
    assert gm.contract_ok(g)
    for bad in (replace(g, a_misalign=1), replace(g, lda=g.lda + 1), replace(g, K=63), replace(g, ldc=127),
                replace(g, alias="A"), replace(g, alias="B")):
        assert not gm.contract_ok(bad)
