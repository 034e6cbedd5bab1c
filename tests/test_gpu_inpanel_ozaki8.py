"""The in-panel update of a two-level outer panel (engine.cu, factor_outer_panel) on the eight-bit kernel, bit for bit
against its exact model (tests/ozaki8_exact_model.py), through ``agp_debug_ozaki8``: the first half's slices (every row
below it) update the second half's 512 columns, a rectangle of rows below the second half plus the lower tiles of its
diagonal block, with the same closed-form walk, at K = 512 (a 1024-wide panel) and K = 1024 (a 2048-wide one), on
persistent and bounded CTAs.  Owned entries must equal the model exactly; every other element of the C buffer must be
untouched."""
import ctypes as C

import numpy as np
import pytest

import ozaki_exact_model as om
import ozaki8_exact_model as o8

pytestmark = pytest.mark.gpu

BN = om.tile_width(6)
PAD = 37


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _same_bits(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert bad.size == 0, "%d elements differ, first at %s: got %r want %r" % (bad.size, bad[:8], got[bad[:4]], want[bad[:4]])


@pytest.mark.parametrize("K", [512, 1024])
@pytest.mark.parametrize("M", [1280, 1280 - 37, 512])
@pytest.mark.parametrize("chunk", [None, "1", "8"])
def test_in_panel_update(ag, monkeypatch, K, M, chunk):
    """N = 512 columns of the second half; M rows from its first row down (M = 512: the last panel, only the diagonal
    block; a ragged M: rows past it untouched)"""
    import torch
    monkeypatch.delenv("AGP_OZAKI_CHUNK_TEST", raising=False)
    if chunk:
        monkeypatch.setenv("AGP_OZAKI_CHUNK_TEST", chunk)
    rng = np.random.default_rng(K + M)
    N, ldc = 512, M + 3
    P = rng.standard_normal((M, K)) * np.ldexp(1.0, rng.integers(-8, 8, (M, 1)))
    Cbuf = rng.random(ldc * N + PAD) + 0.25
    ws = o8.Workspace(K, M).put(P)
    owned = om.owned_lower(M, N, BN)
    assert owned.any() and not owned.all()
    want = o8.expected_update(ws, Cbuf, ldc, M, N, -1.0, 0, om.column_rows(N, BN, 0), owned)
    eng = ag.engine()
    Cd, Pd = _dev(Cbuf), _dev(P.T)
    torch.cuda.synchronize()
    rc = eng.L.agp_debug_ozaki8(eng.h, C.c_void_p(Cd.data_ptr()), ldc, C.c_void_p(Pd.data_ptr()), 0, M, M, None, 0, 0,
                                M, N, K, -1.0, 0, 0, 0, 0)
    eng.check(rc)
    _same_bits(Cd.cpu().numpy(), want)
