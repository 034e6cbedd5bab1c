"""Why the bit-exact tests of the eight-bit update kernel may model it with 128 x 32 tiles (BN = om.tile_width(6) = 32)
although it runs 128 x 64 tiles: for every shape and offset agp_debug_ozaki8 accepts (N a multiple of 128, row and
column offsets in whole 128-row blocks, a block-cyclic stride and width in multiples of 128), both tile widths write
exactly the same elements of C, each once, and map every column to the same panel row.  Checked on the kernel's two
walks -- the closed-form, L2-blocked lower walk (oz_tile) and the strip table -- and against the exact model's
owned_lower / owned_table / column_rows.  The arithmetic of an element does not depend on its tile, so the same
elements with the same column rows give the same bits."""
import numpy as np
import pytest

import ozaki_exact_model as om
import test_tile_enumeration as te

BNS = (32, 64)


def _closed_form(M, N, BN, b_off):
    """written-count mask and column -> panel row map of the closed-form walk (a_off == b_off, identity column map)"""
    R = om.BM // BN
    nbi, nbj = -(-M // om.BM), -(-N // BN)
    hits = np.zeros((M, N), np.int32)
    col_row = np.full(N, -1, np.int64)
    for t in range(te.n_slots(nbi, nbj, R)):
        bi, bj, ok = te.oz_tile(t, nbi, nbj, R)
        if not ok:
            continue
        hits[bi * om.BM:(bi + 1) * om.BM, bj * BN:(bj + 1) * BN] += 1
        cols = np.arange(bj * BN, min(N, (bj + 1) * BN))
        col_row[cols] = bj * BN + b_off + (cols - bj * BN)
    return hits, col_row


def _table(M, N, BN, stride, bw, b_off, a_off):
    """the same for the strip-table walk (block-cyclic column map, a_off != b_off)"""
    nbi, nbj = -(-M // om.BM), -(-N // BN)
    start, bimin, n = te.strip_table(nbi, nbj, stride, bw, b_off, a_off, BN)
    hits = np.zeros((M, N), np.int32)
    col_row = np.full(N, -1, np.int64)
    bwe = bw or om.BM
    for t in range(n):
        bi, bj = te.tab_decode(t, start, bimin, nbj)
        hits[bi * om.BM:(bi + 1) * om.BM, bj * BN:(bj + 1) * BN] += 1
        n0 = bj * BN
        brow = ((n0 // bwe) * stride + n0 % bwe if stride else n0) + b_off
        cols = np.arange(n0, min(N, n0 + BN))
        col_row[cols] = brow + (cols - n0)
    return hits, col_row


@pytest.mark.parametrize("M,N,off", [(128, 128, 0), (200, 128, 0), (1000, 640, 256), (1152, 1024, 0), (2176, 2048, 128),
                                     (2304, 2304, 0), (4224, 4096, 0), (1300, 2560, 384)])
def test_closed_form_walk(M, N, off):
    got = {BN: _closed_form(M, N, BN, off) for BN in BNS}
    for BN in BNS:
        hits, col_row = got[BN]
        assert hits.max() == 1
        assert np.array_equal(hits == 1, om.owned_lower(M, N, BN))
        seen = col_row >= 0  # columns no row tile reaches (N > M) are never mapped
        assert np.array_equal(col_row[seen], om.column_rows(N, BN, off)[seen])
    assert np.array_equal(got[32][0], got[64][0])
    assert np.array_equal(got[32][1], got[64][1])


@pytest.mark.parametrize("M,N,stride,bw,b_off,a_off", [
    (768, 640, 0, 0, 512, 512),          # identity map with offsets, through the table
    (1536, 512, 512, 256, 256, 128),     # block-cyclic, a_off != b_off
    (1408, 512, 512, 128, 0, 128),       # bw = 128
    (2304, 1024, 1024, 512, 256, 256),   # bw = 512
    (1000, 768, 384, 128, 128, 0),
    (1536, 512, 768, 256, 0, 0)])
def test_strip_table_walk(M, N, stride, bw, b_off, a_off):
    got = {BN: _table(M, N, BN, stride, bw, b_off, a_off) for BN in BNS}
    for BN in BNS:
        hits, col_row = got[BN]
        assert hits.max() == 1
        assert np.array_equal(hits == 1, om.owned_table(M, N, BN, b_off, a_off, stride, bw))
        seen = col_row >= 0
        assert np.array_equal(col_row[seen], om.column_rows(N, BN, b_off, stride, bw)[seen])
    assert np.array_equal(got[32][0], got[64][0])
    assert np.array_equal(got[32][1], got[64][1])

