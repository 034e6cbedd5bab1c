"""The 128 x 64 tile of the eight-bit update kernel (``ozaki8_update_kernel``: both operands from shared memory, 21
m64n64k32 MMAs per chunk) bit for bit against its exact model (tests/ozaki8_exact_model.py) through
``agp_debug_ozaki8``, on the edges the wider tile creates: a partial last row tile, one column-tile pair (N = 128) and an
odd number of them (N = 640), block-cyclic column maps with bw = 128 and 512, bounded CTAs whose tile count is not a
multiple of the CTA size, K from two chunks (fewer than the ring's stages) to 16 384, staged and unstaged drains.
Owned entries must equal the model exactly; every other element of the C buffer must be untouched."""
import ctypes as C

import numpy as np
import pytest

import ozaki_exact_model as om
import ozaki8_exact_model as o8

pytestmark = pytest.mark.gpu

BN = 64
PAD = 29
# persistent CTAs, then bounded CTAs of 3 and 5 tiles (AGP_OZAKI_CHUNK_TEST counts 128 x 32 tiles, two per 128 x 64 tile)
CTA_ENVS = [{}, {"AGP_OZAKI_CHUNK_TEST": "6"}, {"AGP_OZAKI_CHUNK_TEST": "10"}]


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def _set_env(monkeypatch, env):
    monkeypatch.delenv("AGP_OZAKI_CHUNK_TEST", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _rows(rng, m, K):
    return rng.standard_normal((m, K)) * np.ldexp(1.0, rng.integers(-8, 8, (m, 1)))


def _c_buffer(rng, ldc, N):
    return rng.random(ldc * N + PAD) + 0.25


def _call(ag, Cbuf, ldc, A, M, N, K, sign, B=None, m_panel=0, stride=0, bw=0, b_off=0, a_off=0):
    import torch
    eng = ag.engine()
    Cd, Ad = _dev(Cbuf), _dev(A.T)
    Bd = _dev(B) if B is not None else None
    torch.cuda.synchronize()
    rc = eng.L.agp_debug_ozaki8(eng.h, _ptr(Cd), ldc, _ptr(Ad), 0, A.shape[0], m_panel, _ptr(Bd) if Bd is not None else None,
                                1, K, M, N, K, sign, stride, bw, b_off, a_off)
    eng.check(rc)
    return Cd.cpu().numpy()


def _same_bits(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert bad.size == 0, "%d elements differ, first at %s: got %r want %r" % (bad.size, bad[:8], got[bad[:4]], want[bad[:4]])


def _gemm_case(rng, M, N, K, ldc, sign):
    A, B = _rows(rng, M, K), _rows(rng, N, K)
    Cbuf = _c_buffer(rng, ldc, N)
    m_pad = om.ceil128(M)
    ws = o8.Workspace(K, m_pad + om.ceil128(N)).put(A).put(B, m_pad)
    want = o8.expected_update(ws, Cbuf, ldc, M, N, sign, 0, om.column_rows(N, BN, m_pad), np.ones((M, N), bool))
    return A, B, Cbuf, want


# ---- rectangular walk: row and column edges x drains x CTA forms -------------------------------------------------------
@pytest.mark.parametrize("M,N", [(200, 128), (1000, 640), (256, 640)])
@pytest.mark.parametrize("drain", ["staged", "unstaged"])
def test_row_and_column_edges(ag, monkeypatch, M, N, drain):
    """full tiles stage their C block when ldc keeps every column 16-byte aligned; an odd ldc sends every tile through
    the guarded global drain.  M = 200 and 1000 end in a partial row tile (always the global drain); N = 128 is one
    column-tile pair, N = 640 five"""
    rng = np.random.default_rng(M + N + len(drain))
    K, sign = 256, -1.0
    ldc = M + (0 if drain == "staged" else 1)
    A, B, Cbuf, want = _gemm_case(rng, M, N, K, ldc, sign)
    for env in CTA_ENVS:
        _set_env(monkeypatch, env)
        _same_bits(_call(ag, Cbuf, ldc, A, M, N, K, sign, B=B), want)


# ---- K: fewer chunks than stages, a few rounds of the ring, the largest accepted -------------------------------------
@pytest.mark.parametrize("K", [64, 512, 16384])
def test_k_lengths(ag, monkeypatch, K):
    rng = np.random.default_rng(K)
    M, N, ldc = 384, 256, 384
    A, B, Cbuf, want = _gemm_case(rng, M, N, K, ldc, 1.0)
    for env in CTA_ENVS[:2]:
        _set_env(monkeypatch, env)
        _same_bits(_call(ag, Cbuf, ldc, A, M, N, K, 1.0, B=B), want)


# ---- lower and strip-table walks over one panel ------------------------------------------------------------------------
@pytest.mark.parametrize("m_panel,M,N,stride,bw,b_off,a_off", [
    (1152, 1152, 640, 0, 0, 0, 0),          # closed-form lower walk, partial super-block
    (1280, 1000, 640, 0, 0, 256, 256),      # closed-form walk with offsets, partial last row tile
    (1792, 1408, 512, 512, 128, 0, 128),    # block-cyclic strip table, bw = 128
    (2560, 2304, 1024, 1024, 512, 256, 256)])  # block-cyclic strip table, bw = 512
def test_panel_walks(ag, monkeypatch, m_panel, M, N, stride, bw, b_off, a_off):
    rng = np.random.default_rng(m_panel + bw)
    K, sign = 128, -1.0
    ldc = M + (M & 1)  # an even ldc: full tiles stage, the partial row tile drains from global memory
    P = _rows(rng, m_panel, K)
    Cbuf = _c_buffer(rng, ldc, N)
    ws = o8.Workspace(K, m_panel).put(P)
    cols = om.column_rows(N, BN, b_off, stride, bw)
    owned = om.owned_lower(M, N, BN) if stride == 0 and a_off == b_off else om.owned_table(M, N, BN, b_off, a_off, stride, bw)
    assert owned.any() and not owned.all()
    want = o8.expected_update(ws, Cbuf, ldc, M, N, sign, a_off, cols, owned)
    for env in CTA_ENVS:
        _set_env(monkeypatch, env)
        _same_bits(_call(ag, Cbuf, ldc, P, M, N, K, sign, m_panel=m_panel, stride=stride, bw=bw, b_off=b_off, a_off=a_off),
                   want)
