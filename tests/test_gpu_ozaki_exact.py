"""The int8-slice update kernel bit for bit against its exact model (tests/ozaki_exact_model.py), through the three debug
entries: every compiled instantiation (fp64 C with 4..8 slices, fp32 C with 3..5), both drains (staged C block and
guarded global loads, alone and mixed in one launch), both epilogues (int32 pairs and plain int64 words), persistent and
bounded CTAs, the K edges, the three tile walks, the edges of the exponent range and non-finite operands.  Owned
entries must equal the model exactly; every other element of the C buffer -- tiles above the diagonal, rows from M to
ldc, the elements just outside C -- must be untouched."""
import ctypes as C

import numpy as np
import pytest

import ozaki_exact_model as om

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
PAD = 37                                             # guard elements after C in every buffer
ENVS = [{}, {"AGP_OZAKI_EPI": "0"}, {"AGP_OZAKI_CHUNK_TEST": "1"}, {"AGP_OZAKI_CHUNK_TEST": "4"},
        {"AGP_OZAKI_EPI": "0", "AGP_OZAKI_CHUNK_TEST": "1"}, {"AGP_OZAKI_EPI": "0", "AGP_OZAKI_CHUNK_TEST": "4"}]


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def _store(P, dt, kmajor):
    """device storage of the rows of P: row-contiguous (element (r, k) at [r + k * ld]) or k-major ([k + r * ld])"""
    P = P.astype(dt)
    return (_dev(P), P.shape[1]) if kmajor else (_dev(P.T), P.shape[0])


def _c_buffer(rng, ldc, N, cdt, base=0):
    """column-major C (ldc x N) at element `base` of a buffer with PAD guard elements after it"""
    return (rng.random(base + ldc * N + PAD) + 0.25).astype(cdt)


def _set_env(monkeypatch, env):
    for k in ("AGP_OZAKI_EPI", "AGP_OZAKI_CHUNK_TEST"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)       # the launcher reads both per call


def _gemm(ag, Cbuf, ldc, base, A, adt, akm, B, bdt, bkm, N, K, S, sign):
    import torch
    eng = ag.engine()
    Cd = _dev(Cbuf)
    Ad, lda = _store(A, adt, akm)
    Bd, ldb = _store(B, bdt, bkm) if B is not None else (None, 0)
    torch.cuda.synchronize()
    rc = eng.L.agp_debug_ozaki_gemm(eng.h, _ptr(Cd, base), int(Cbuf.dtype == F32), ldc, _ptr(Ad), int(adt == F32), int(akm), lda,
                                    A.shape[0], _ptr(Bd) if Bd is not None else None, int(bdt == F32), int(bkm), ldb, N, K, S, sign)
    eng.check(rc)
    return Cd.cpu().numpy()


def _model_gemm(Cbuf, ldc, base, A, B, N, K, S, sign, pair32, adt=F64, bdt=F64):
    """what agp_debug_ozaki_gemm computes: A rows at 0, B rows from the next multiple of 128 (rectangular walk), or
    without B the lower tiles of A A'"""
    M, BN = A.shape[0], om.tile_width(S)
    m_pad = om.ceil128(M)
    ws = om.Workspace(S, K, m_pad + (om.ceil128(N) if B is not None else 0))
    ws.put(A.astype(adt))
    if B is not None:
        ws.put(B.astype(bdt), m_pad)
        cols, owned = om.column_rows(N, BN, m_pad), np.ones((M, N), bool)
    else:
        cols, owned = om.column_rows(N, BN, 0), om.owned_lower(M, N, BN)
    return om.expected_update(ws, Cbuf, ldc, M, N, sign, 0, cols, owned, pair32, Cbuf.dtype == F32, base)


def _syrk(ag, Cbuf, ldc, P, N, K, S, lower):
    import torch
    eng = ag.engine()
    Cd, (Pd, lda) = _dev(Cbuf), _store(P, F64, 0)
    torch.cuda.synchronize()
    eng.check(eng.L.agp_debug_ozaki_syrk(eng.h, _ptr(Cd), ldc, _ptr(Pd), lda, P.shape[0], N, K, S, int(lower)))
    return Cd.cpu().numpy()


def _model_syrk(Cbuf, ldc, P, N, K, S, lower, pair32):
    M, BN = P.shape[0], om.tile_width(S)
    ws = om.Workspace(S, K, M).put(P)
    owned = om.owned_lower(M, N, BN) if lower else np.ones((M, N), bool)
    return om.expected_update(ws, Cbuf, ldc, M, N, -1.0, 0, om.column_rows(N, BN, 0), owned, pair32, False)


def _same_bits(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    u = np.uint32 if got.dtype == F32 else np.uint64
    bad = np.nonzero(got.view(u) != want.view(u))[0]
    assert bad.size == 0, "%d elements differ, first at %s: got %r want %r" % (bad.size, bad[:8], got[bad[:4]], want[bad[:4]])


def _rows(rng, m, K, lo=-8, hi=8):
    return rng.standard_normal((m, K)) * np.ldexp(1.0, rng.integers(lo, hi, (m, 1)))


# ---- every instantiation -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,cdt,adt,bdt,akm,bkm,sign", [
    (4, F64, F32, F64, 0, 1, -1.0), (5, F64, F64, F64, 1, 0, 1.0), (6, F64, F64, F32, 0, 0, -1.0),
    (7, F64, F64, F64, 1, 1, -1.0), (8, F64, F32, F32, 0, 1, 1.0),
    (3, F32, F32, F32, 1, 0, -1.0), (4, F32, F64, F32, 0, 0, 1.0), (5, F32, F32, F64, 1, 1, -1.0)])
def test_every_instantiation(ag, S, cdt, adt, bdt, akm, bkm, sign):
    """300 x 256 with aligned C: staged full tiles and guarded partial ones in one launch"""
    rng = np.random.default_rng(S * 10 + (cdt == F32))
    M, N, K, ldc = 300, 256, 192, 304
    A, B = _rows(rng, M, K), _rows(rng, N, K)
    Cbuf = _c_buffer(rng, ldc, N, cdt)
    want = _model_gemm(Cbuf, ldc, 0, A, B, N, K, S, sign, om.pair32_used(S, K), adt, bdt)
    _same_bits(_gemm(ag, Cbuf, ldc, 0, A, adt, akm, B, bdt, bkm, N, K, S, sign), want)


# ---- drain paths x epilogues x CTA forms ------------------------------------------------------------------------------
DRAINS = {  # name: (M, ldc(M, itemsize), base)
    "staged": ([256], lambda M, w: M, 0),
    "odd_ldc": ([256], lambda M, w: M + 1, 0),
    "mixed": ([1, 127, 129, 1000], lambda M, w: -(-M // (16 // w)) * (16 // w), 0),
    "base_plus_one": ([256], lambda M, w: M, 1),
}


@pytest.mark.parametrize("S,cdt", [(7, F64), (4, F32)])
@pytest.mark.parametrize("path", sorted(DRAINS))
def test_drain_paths(ag, monkeypatch, path, S, cdt):
    Ms, ldc_of, base = DRAINS[path]
    rng = np.random.default_rng(len(path) + S)
    K, N = 256, 256
    for M in Ms:
        ldc = ldc_of(M, np.dtype(cdt).itemsize)
        A, B = _rows(rng, M, K), _rows(rng, N, K)
        Cbuf = _c_buffer(rng, ldc, N, cdt, base)
        want = _model_gemm(Cbuf, ldc, base, A, B, N, K, S, 1.0, om.pair32_used(S, K))
        for env in ENVS:
            _set_env(monkeypatch, env)
            _same_bits(_gemm(ag, Cbuf, ldc, base, A, F64, 0, B, F64, 1, N, K, S, 1.0), want)


@pytest.mark.parametrize("lower", [True, False])
def test_partial_column_strips(ag, monkeypatch, lower):
    """syrk with N = 100: the last 32-column strip is partial; aligned C, so full tiles are staged"""
    rng = np.random.default_rng(3)
    M, N, K, S, ldc = 300, 100, 128, 6, 300
    P = _rows(rng, M, K)
    Cbuf = _c_buffer(rng, ldc, N, F64)
    want = _model_syrk(Cbuf, ldc, P, N, K, S, lower, True)
    for env in ENVS:
        _set_env(monkeypatch, env)
        _same_bits(_syrk(ag, Cbuf, ldc, P, N, K, S, lower), want)


# ---- K edges, with digits near their bounds ---------------------------------------------------------------------------
@pytest.mark.parametrize("K", [64, 512, 576, 4096, 32768])
@pytest.mark.parametrize("near", [False, True])
def test_k_edges_fp64(ag, K, near):
    """fp64 C through syrk (160 rows: one full and one partial row tile, two 32-column strips); S = 7, and S = 8 (one
    fragment buffer) at K = 4096"""
    rng = np.random.default_rng(K + near)
    M, N, ldc = 160, 64, 160
    for S in ([7, 8] if K == 4096 else [7]):
        P = om.digits_to_values(om.near_bound_digits(rng, S, M, K)) if near else _rows(rng, M, K)
        Cbuf = _c_buffer(rng, ldc, N, F64)
        want = _model_syrk(Cbuf, ldc, P, N, K, S, False, om.pair32_used(S, K))
        _same_bits(_syrk(ag, Cbuf, ldc, P, N, K, S, False), want)


@pytest.mark.parametrize("K", [64, 576, 32768])
@pytest.mark.parametrize("S", [4, 5])
def test_k_edges_fp32_c(ag, K, S):
    """fp32 C at the K edges with near-bound digits in fp64 operands (fp32 operands cannot hold them at S = 5)"""
    rng = np.random.default_rng(K * S)
    M, N, ldc = 130, 128, 132
    A = om.digits_to_values(om.near_bound_digits(rng, S, M, K))
    B = om.digits_to_values(om.near_bound_digits(rng, S, N, K))
    Cbuf = _c_buffer(rng, ldc, N, F32)
    want = _model_gemm(Cbuf, ldc, 0, A, B, N, K, S, -1.0, om.pair32_used(S, K))
    _same_bits(_gemm(ag, Cbuf, ldc, 0, A, F64, 1, B, F64, 0, N, K, S, -1.0), want)


# ---- tile walks ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [2304, 4224])
def test_lower_walk_across_super_blocks(ag, N):
    """the closed-form, L2-blocked lower walk on the Cholesky's shape: M = N + 128 border rows"""
    rng = np.random.default_rng(N)
    M, K, S = N + 128, 64, 5
    P = _rows(rng, M, K)
    Cbuf = _c_buffer(rng, M, N, F64)
    _same_bits(_syrk(ag, Cbuf, M, P, N, K, S, True), _model_syrk(Cbuf, M, P, N, K, S, True, True))


def test_lower_walk_tall(ag):
    """more super-block rows than columns (the walk's second branch), fp32 C without B"""
    rng = np.random.default_rng(11)
    M, N, K, S, ldc = 2200, 128, 64, 4, 2200
    A = _rows(rng, M, K)
    Cbuf = _c_buffer(rng, ldc, N, F32)
    _same_bits(_gemm(ag, Cbuf, ldc, 0, A, F32, 0, None, F32, 0, N, K, S, -1.0),
               _model_gemm(Cbuf, ldc, 0, A, None, N, K, S, -1.0, False, F32))


@pytest.mark.parametrize("m_panel,M,N,S,stride,bw,b_off,a_off", [
    (1280, 768, 640, 7, 0, 0, 512, 512),          # the rest update of cholesky_inplace: closed-form walk, offsets
    (1664, 1536, 512, 6, 512, 256, 256, 128),     # block-cyclic strip table, a_off != b_off
    (1536, 1536, 512, 8, 768, 256, 0, 0)])
def test_mapped_walks(ag, m_panel, M, N, S, stride, bw, b_off, a_off):
    import torch
    eng = ag.engine()
    rng = np.random.default_rng(m_panel + S)
    K, ldc = 128, M + 3
    P = _rows(rng, m_panel, K)
    Cbuf = _c_buffer(rng, ldc, N, F64)
    BN = om.tile_width(S)
    ws = om.Workspace(S, K, m_panel).put(P)
    cols = om.column_rows(N, BN, b_off, stride, bw)
    owned = om.owned_lower(M, N, BN) if stride == 0 and a_off == b_off else om.owned_table(M, N, BN, b_off, a_off, stride, bw)
    want = om.expected_update(ws, Cbuf, ldc, M, N, -1.0, a_off, cols, owned, True, False)
    Cd, (Pd, lda) = _dev(Cbuf), _store(P, F64, 0)
    torch.cuda.synchronize()
    eng.check(eng.L.agp_debug_ozaki_syrk_map(eng.h, _ptr(Cd), ldc, _ptr(Pd), lda, m_panel, M, N, K, S, stride, bw, b_off, a_off))
    _same_bits(Cd.cpu().numpy(), want)
    assert owned.any() and not owned.all()


# ---- exponent range -------------------------------------------------------------------------------------------------------
def _check_exact_bound(got_flat, Cbuf, ldc, A, B, S, sign, picks):
    cf = Cbuf.dtype == F32
    ea, eb = om.row_exponents(A)[0], om.row_exponents(B)[0]
    K = A.shape[1]
    from fractions import Fraction
    for i, j in picks:
        g = got_flat[i + j * ldc]
        ex = om.exact_entry(Cbuf[i + j * ldc], A[i], B[j], sign)
        assert abs(Fraction(float(g)) - ex) <= om.result_bound(S, ea[i], eb[j], K, g, cf), (i, j)


@pytest.mark.parametrize("S,cdt,odt", [(7, F64, F64), (4, F32, F32), (7, F64, F32)])
def test_exponent_edges(ag, S, cdt, odt):
    """rows scaled 2^-1000 .. 2^990, an all-zero row, subnormal-only rows (C_old = 0 there, so their products are the
    result) and a normal row with entries 2^-1074; for fp32 operands, rows of fp32 subnormals and rows with subnormal
    entries.  Bit-exact with the model and within the exact bound."""
    rng = np.random.default_rng(S + (odt == F32))
    M, N, K, ldc = 160, 128, 128, 160
    if odt == F64:
        A = rng.standard_normal((M, K)) * np.ldexp(1.0, rng.integers(-1000, 990, (M, 1)))
        A[2:6] = rng.standard_normal((4, K)) * 1e-310                     # subnormal only
        A[6, ::3] = 5e-324
    else:
        A = (rng.standard_normal((M, K)) * np.ldexp(1.0, rng.integers(-60, 60, (M, 1)))).astype(F32).astype(F64)
        A[2:6] = (rng.standard_normal((4, K)) * 1e-40).astype(F32)        # fp32 subnormal only
        A[6:10, ::2] = (rng.standard_normal((4, K // 2)) * 1e-42).astype(F32)   # subnormal entries in normal rows
    A[1] = 0.0
    B = rng.standard_normal((N, K)) * np.ldexp(1.0, rng.integers(-8, 8, (N, 1)))
    if odt == F32:
        B = B.astype(F32).astype(F64)
    Cbuf = _c_buffer(rng, ldc, N, cdt)
    for j in range(N):
        Cbuf[2 + j * ldc:11 + j * ldc] = 0.0
    want = _model_gemm(Cbuf, ldc, 0, A, B, N, K, S, -1.0, om.pair32_used(S, K), odt, odt)
    got = _gemm(ag, Cbuf, ldc, 0, A, odt, 0, B, odt, 1, N, K, S, -1.0)
    _same_bits(got, want)
    picks = [(i, j) for i in range(8) for j in (0, 1, 5, N - 1)] + [(40, 7), (M - 1, N - 1)]
    _check_exact_bound(got, Cbuf, ldc, A, B, S, -1.0, picks)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("where", ["A", "B", "syrk"])
def test_non_finite_operands(ag, bad, where):
    """one NaN or +-Inf entry: exactly the entries an fp64 reference makes non-finite are non-finite, the rest is
    bit-exact (BLAS semantics instead of a silently dropped NaN or wrapped digits)"""
    rng = np.random.default_rng(17)
    M, N, K, S, ldc = 200, 128, 128, 7, 200
    A, B = _rows(rng, M, K), _rows(rng, N, K)
    Cbuf = _c_buffer(rng, ldc, N, F64)
    if where == "syrk":
        A[70, 33] = bad
        got = _syrk(ag, Cbuf, ldc, A, N, K, S, True)
        want = _model_syrk(Cbuf, ldc, A, N, K, S, True, True)
        owned = om.owned_lower(M, N, om.tile_width(S))
        with np.errstate(invalid="ignore", over="ignore"):
            ref = Cbuf[:ldc * N].reshape(N, ldc).T[:M].copy() - A @ A[:N].T
    else:
        (A if where == "A" else B)[5, 17] = bad
        got = _gemm(ag, Cbuf, ldc, 0, A, F64, 0, B, F64, 0, N, K, S, 1.0)
        want = _model_gemm(Cbuf, ldc, 0, A, B, N, K, S, 1.0, True)
        owned = np.ones((M, N), bool)
        with np.errstate(invalid="ignore", over="ignore"):
            ref = Cbuf[:ldc * N].reshape(N, ldc).T[:M].copy() + A @ B.T
    g = got[:ldc * N].reshape(N, ldc).T[:M]
    assert np.array_equal(np.isfinite(g)[owned], np.isfinite(ref)[owned])
    assert (~np.isfinite(g)).sum() > 0
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin)
    _same_bits(got[fin], want[fin])


# ---- argument checks --------------------------------------------------------------------------------------------------------
def test_debug_entries_reject_bad_arguments(ag):
    import torch
    from agp_b200 import _cabi
    eng = ag.engine()
    Cd = torch.zeros(512 * 512, dtype=torch.float64, device="cuda")
    Pd = torch.zeros(512 * 128, dtype=torch.float64, device="cuda")
    c, p = _ptr(Cd), _ptr(Pd)
    L = eng.L
    torch.cuda.synchronize()
    for S in (3, 4):   # fp64 C has no 3- or 4-slice kernel
        assert L.agp_debug_ozaki_syrk(eng.h, c, 256, p, 256, 256, 128, 128, S, 1) == _cabi.AGP_ERR_UNSUPPORTED
        assert L.agp_debug_ozaki_syrk_map(eng.h, c, 256, p, 256, 256, 256, 128, 128, S, 0, 0, 0, 0) == _cabi.AGP_ERR_UNSUPPORTED
    assert L.agp_debug_ozaki_syrk(eng.h, c, 256, p, 256, 128, 256, 128, 7, 1) == _cabi.AGP_ERR_INVALID        # N > M
    assert L.agp_debug_ozaki_gemm(eng.h, c, 0, 256, p, 0, 0, 256, 128, None, 0, 0, 0, 256, 128, 7, -1.0) == _cabi.AGP_ERR_INVALID
    # columns mapped past the panel: a strip table that would read rows nobody sliced
    assert L.agp_debug_ozaki_syrk_map(eng.h, c, 256, p, 256, 256, 256, 256, 128, 7, 512, 128, 0, 0) == _cabi.AGP_ERR_INVALID
    assert L.agp_debug_ozaki_syrk_map(eng.h, c, 256, p, 256, 256, 256, 128, 128, 7, 0, 0, 256, 0) == _cabi.AGP_ERR_INVALID
    assert L.agp_debug_ozaki_syrk_map(eng.h, c, 256, p, 256, 256, 256, 128, 128, 7, 0, 0, 0, 128) == _cabi.AGP_ERR_INVALID
    assert float(Cd.abs().max()) == 0.0                                                       # nothing ran
    assert L.agp_debug_ozaki_syrk(eng.h, c, 256, p, 256, 256, 128, 128, 7, 1) == 0            # and the context still works
