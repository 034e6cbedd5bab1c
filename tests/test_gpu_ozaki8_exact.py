"""The eight-bit format of the int8-slice update (six balanced 8-bit digits, ``ozaki8_update_kernel``) bit for bit against
its exact model (tests/ozaki8_exact_model.py), through ``agp_debug_ozaki8``: the three tile walks, both drains (staged C
block and guarded global loads, alone and mixed in one launch), persistent and bounded CTAs, K from one chunk pair to the
largest accepted (16384) and its rejection above, the edges of the exponent range and non-finite operands.  Owned
entries must equal the model exactly; every other element of the C buffer must be untouched."""
import ctypes as C

import numpy as np
import pytest

import ozaki_exact_model as om
import ozaki8_exact_model as o8

pytestmark = pytest.mark.gpu

PAD = 37
BN = om.tile_width(6)
CTA_ENVS = [{}, {"AGP_OZAKI_CHUNK_TEST": "1"}, {"AGP_OZAKI_CHUNK_TEST": "4"}]


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def _store(P, kmajor):
    return (_dev(P), P.shape[1]) if kmajor else (_dev(P.T), P.shape[0])


def _c_buffer(rng, ldc, N, base=0):
    return rng.random(base + ldc * N + PAD) + 0.25


def _set_env(monkeypatch, env):
    monkeypatch.delenv("AGP_OZAKI_CHUNK_TEST", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _run(ag, Cbuf, ldc, A, M, N, K, sign, base=0, akm=0, B=None, bkm=0, m_panel=0, stride=0, bw=0, b_off=0, a_off=0):
    """agp_debug_ozaki8; returns (status, C buffer after the call)"""
    import torch
    eng = ag.engine()
    Cd = _dev(Cbuf)
    Ad, lda = _store(A, akm)
    Bd, ldb = _store(B, bkm) if B is not None else (None, 0)
    torch.cuda.synchronize()
    rc = eng.L.agp_debug_ozaki8(eng.h, _ptr(Cd, base), ldc, _ptr(Ad), akm, lda, m_panel, _ptr(Bd) if Bd is not None else None,
                                bkm, ldb, M, N, K, sign, stride, bw, b_off, a_off)
    return rc, Cd.cpu().numpy()


def _gemm(ag, Cbuf, ldc, A, B, N, K, sign, base=0, akm=0, bkm=1):
    rc, out = _run(ag, Cbuf, ldc, A, A.shape[0], N, K, sign, base, akm, B, bkm)
    ag.engine().check(rc)
    return out


def _model_gemm(Cbuf, ldc, A, B, N, K, sign, base=0):
    M = A.shape[0]
    m_pad = om.ceil128(M)
    ws = o8.Workspace(K, m_pad + om.ceil128(N)).put(A).put(B, m_pad)
    return o8.expected_update(ws, Cbuf, ldc, M, N, sign, 0, om.column_rows(N, BN, m_pad), np.ones((M, N), bool), base)


def _panel(ag, Cbuf, ldc, P, M, N, K, sign, stride=0, bw=0, b_off=0, a_off=0):
    rc, out = _run(ag, Cbuf, ldc, P, M, N, K, sign, m_panel=P.shape[0], stride=stride, bw=bw, b_off=b_off, a_off=a_off)
    ag.engine().check(rc)
    return out


def _model_panel(Cbuf, ldc, P, M, N, K, sign, stride=0, bw=0, b_off=0, a_off=0):
    ws = o8.Workspace(K, P.shape[0]).put(P)
    cols = om.column_rows(N, BN, b_off, stride, bw)
    owned = om.owned_lower(M, N, BN) if stride == 0 and a_off == b_off else om.owned_table(M, N, BN, b_off, a_off, stride, bw)
    return o8.expected_update(ws, Cbuf, ldc, M, N, sign, a_off, cols, owned), owned


def _same_bits(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert bad.size == 0, "%d elements differ, first at %s: got %r want %r" % (bad.size, bad[:8], got[bad[:4]], want[bad[:4]])


def _rows(rng, m, K, lo=-8, hi=8):
    return rng.standard_normal((m, K)) * np.ldexp(1.0, rng.integers(lo, hi, (m, 1)))


# ---- rectangular walk: operand layouts x drains x CTA forms -----------------------------------------------------------
DRAINS = {  # name: (M values, ldc(M), base)
    "staged": ([256], lambda M: M, 0),
    "odd_ldc": ([256], lambda M: M + 1, 0),
    "mixed": ([1, 127, 129, 1000], lambda M: M + (M & 1), 0),
    "base_plus_one": ([256], lambda M: M, 1),
}


@pytest.mark.parametrize("path", sorted(DRAINS))
def test_drain_paths_and_cta_forms(ag, monkeypatch, path):
    Ms, ldc_of, base = DRAINS[path]
    rng = np.random.default_rng(len(path))
    K, N = 256, 256
    for M in Ms:
        ldc = ldc_of(M)
        A, B = _rows(rng, M, K), _rows(rng, N, K)
        Cbuf = _c_buffer(rng, ldc, N, base)
        want = _model_gemm(Cbuf, ldc, A, B, N, K, 1.0, base)
        for env in CTA_ENVS:
            _set_env(monkeypatch, env)
            _same_bits(_gemm(ag, Cbuf, ldc, A, B, N, K, 1.0, base), want)


@pytest.mark.parametrize("akm,bkm", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_operand_layouts(ag, akm, bkm):
    rng = np.random.default_rng(10 + 2 * akm + bkm)
    M, N, K, ldc = 300, 256, 192, 304
    A, B = _rows(rng, M, K), _rows(rng, N, K)
    Cbuf = _c_buffer(rng, ldc, N)
    want = _model_gemm(Cbuf, ldc, A, B, N, K, -1.0)
    _same_bits(_gemm(ag, Cbuf, ldc, A, B, N, K, -1.0, akm=akm, bkm=bkm), want)


# ---- K edges, with digits near their bounds ---------------------------------------------------------------------------
@pytest.mark.parametrize("K", [64, 512, 1024, 16384])
@pytest.mark.parametrize("near", [False, True])
def test_k_edges(ag, K, near):
    """160 rows (one full and one partial row tile) against 128 columns; near: aligned digits with |q_0| in [56, 63] and
    tails in [120, 127], so the last diagonal reaches 61 % of the int32 range at K = 16384"""
    rng = np.random.default_rng(K + near)
    M, N, ldc = 160, 128, 160
    if near:
        A, B = (o8.digits_to_values(o8.near_bound_digits(rng, m, K)) for m in (M, N))
    else:
        A, B = _rows(rng, M, K), _rows(rng, N, K)
    Cbuf = _c_buffer(rng, ldc, N)
    _same_bits(_gemm(ag, Cbuf, ldc, A, B, N, K, -1.0), _model_gemm(Cbuf, ldc, A, B, N, K, -1.0))


def test_k_above_the_limit_is_rejected(ag):
    from agp_b200 import _cabi
    rng = np.random.default_rng(1)
    K, M, N = o8.MAX_K + 64, 128, 128
    A, B = _rows(rng, M, K), _rows(rng, N, K)
    Cbuf = _c_buffer(rng, M, N)
    rc, out = _run(ag, Cbuf, M, A, M, N, K, -1.0, B=B, bkm=1)
    assert rc == _cabi.AGP_ERR_UNSUPPORTED
    _same_bits(out, Cbuf)
    P = _rows(rng, M, K)
    rc, out = _run(ag, Cbuf, M, P, M, N, K, -1.0, m_panel=M)
    assert rc == _cabi.AGP_ERR_UNSUPPORTED
    _same_bits(out, Cbuf)


# ---- lower and strip-table walks ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [384, 2304])
def test_lower_walk(ag, monkeypatch, N):
    """the closed-form, L2-blocked lower walk on the Cholesky's shape: M = N + 128 border rows; tiles above the diagonal
    and rows past M untouched"""
    rng = np.random.default_rng(N)
    M, K, ldc = N + 128, 128, N + 131
    P = _rows(rng, M, K)
    Cbuf = _c_buffer(rng, ldc, N)
    want, owned = _model_panel(Cbuf, ldc, P, M, N, K, -1.0)
    assert owned.any() and not owned.all()
    for env in CTA_ENVS[:2]:
        _set_env(monkeypatch, env)
        _same_bits(_panel(ag, Cbuf, ldc, P, M, N, K, -1.0), want)


@pytest.mark.parametrize("m_panel,M,N,stride,bw,b_off,a_off,sign", [
    (1280, 768, 640, 0, 0, 512, 512, -1.0),        # the rest update of cholesky_inplace: closed-form walk, offsets
    (1664, 1536, 512, 512, 256, 256, 128, -1.0),   # block-cyclic strip table, a_off != b_off
    (1536, 1536, 512, 768, 256, 0, 0, 1.0)])
def test_mapped_walks(ag, m_panel, M, N, stride, bw, b_off, a_off, sign):
    rng = np.random.default_rng(m_panel + stride)
    K, ldc = 128, M + 3
    P = _rows(rng, m_panel, K)
    Cbuf = _c_buffer(rng, ldc, N)
    want, owned = _model_panel(Cbuf, ldc, P, M, N, K, sign, stride, bw, b_off, a_off)
    _same_bits(_panel(ag, Cbuf, ldc, P, M, N, K, sign, stride, bw, b_off, a_off), want)
    assert owned.any() and not owned.all()


# ---- exponent range and non-finite operands ------------------------------------------------------------------------------
def test_exponent_edges(ag):
    """rows scaled 2^-1000 .. 2^990, an all-zero row, subnormal-only rows (C_old = 0 there) and a normal row with entries
    2^-1074: bit-exact with the model and within the exact bound"""
    from fractions import Fraction
    rng = np.random.default_rng(3)
    M, N, K, ldc = 160, 128, 128, 160
    A = rng.standard_normal((M, K)) * np.ldexp(1.0, rng.integers(-1000, 990, (M, 1)))
    A[2:6] = rng.standard_normal((4, K)) * 1e-310
    A[6, ::3] = 5e-324
    A[1] = 0.0
    B = _rows(rng, N, K)
    Cbuf = _c_buffer(rng, ldc, N)
    for j in range(N):
        Cbuf[2 + j * ldc:11 + j * ldc] = 0.0
    got = _gemm(ag, Cbuf, ldc, A, B, N, K, -1.0, bkm=0)
    _same_bits(got, _model_gemm(Cbuf, ldc, A, B, N, K, -1.0))
    ea, eb = om.row_exponents(A)[0], om.row_exponents(B)[0]
    for i, j in [(i, j) for i in range(8) for j in (0, 1, 5, N - 1)] + [(40, 7), (M - 1, N - 1)]:
        g = got[i + j * ldc]
        ex = om.exact_entry(Cbuf[i + j * ldc], A[i], B[j], -1.0)
        assert abs(Fraction(float(g)) - ex) <= o8.result_bound(ea[i], eb[j], K, g), (i, j)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("where", ["A", "B", "panel"])
def test_non_finite_operands(ag, bad, where):
    """one NaN or +-Inf entry: exactly the entries an fp64 reference makes non-finite are non-finite, the rest is
    bit-exact"""
    rng = np.random.default_rng(17)
    M, N, K, ldc = 200, 128, 128, 200
    A, B = _rows(rng, M, K), _rows(rng, N, K)
    Cbuf = _c_buffer(rng, ldc, N)
    if where == "panel":
        A[70, 33] = bad
        got = _panel(ag, Cbuf, ldc, A, M, N, K, -1.0)
        want, owned = _model_panel(Cbuf, ldc, A, M, N, K, -1.0)
        with np.errstate(invalid="ignore", over="ignore"):
            ref = Cbuf[:ldc * N].reshape(N, ldc).T[:M].copy() - A @ A[:N].T
    else:
        (A if where == "A" else B)[5, 17] = bad
        got = _gemm(ag, Cbuf, ldc, A, B, N, K, 1.0, bkm=0)
        want = _model_gemm(Cbuf, ldc, A, B, N, K, 1.0)
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
def test_rejects_bad_arguments(ag):
    import torch
    from agp_b200 import _cabi
    eng = ag.engine()
    Cd = torch.zeros(512 * 512, dtype=torch.float64, device="cuda")
    Pd = torch.zeros(512 * 128, dtype=torch.float64, device="cuda")
    c, p = _ptr(Cd), _ptr(Pd)
    L, h, INV = eng.L, eng.h, _cabi.AGP_ERR_INVALID
    torch.cuda.synchronize()
    args = lambda **kw: [kw.get(k, d) for k, d in (("m_panel", 256), ("B", None), ("M", 256), ("N", 256), ("K", 128),
                                                   ("stride", 0), ("bw", 0), ("b_off", 0), ("a_off", 0))]

    def call(m_panel, B, M, N, K, stride, bw, b_off, a_off, ldc=256):
        return L.agp_debug_ozaki8(h, c, ldc, p, 0, 256, m_panel, B, 0, 256, M, N, K, -1.0, stride, bw, b_off, a_off)

    assert call(*args(N=100)) == INV                                   # N not a multiple of 128
    assert call(*args(), ldc=128) == INV                               # ldc < M
    assert call(*args(K=96)) == INV                                    # K not a multiple of 64
    assert call(*args(m_panel=128)) == INV                             # columns past the panel
    assert call(*args(stride=512, bw=128)) == INV
    assert call(*args(b_off=256)) == INV
    assert call(*args(a_off=128)) == INV
    assert call(*args(b_off=64)) == INV                                # offsets in whole 128-row blocks
    assert call(*args(B=p, m_panel=0, a_off=128)) == INV               # a product with B takes no offsets
    assert float(Cd.abs().max()) == 0.0                                # nothing ran
    assert call(*args()) == 0                                          # and the context still works
