"""Host-side mirrors of the tile enumerations the persistent int8-slice trailing-update kernel uses
(csrc/umma_ozaki.cu: oz_tile, and the per-strip table of launch_syrk_wgmma).  Output tiles are 128 rows x BN columns,
BN = 64 for up to 4 slices and 32 above (R = 128 / BN column tiles per row tile).  They must visit every tile of the
lower triangle exactly once -- a wrong map would silently skip or double-apply a rank-K update."""
import math

import pytest

SB = 16  # OZ_SB


def oz_tile(t, nbi, nbj, R):
    per = SB * R * SB
    sb, w = divmod(t, per)
    nJ = (nbj + R * SB - 1) // (R * SB)
    t_full = nJ * (nJ + 1) // 2
    if sb < t_full:
        I = int((math.sqrt(8.0 * sb + 1.0) - 1.0) * 0.5)
        while (I + 1) * (I + 2) // 2 <= sb:
            I += 1
        while I * (I + 1) // 2 > sb:
            I -= 1
        Jc = sb - I * (I + 1) // 2
    else:
        r = sb - t_full
        I, Jc = nJ + r // nJ, r % nJ
    bi = I * SB + w // (R * SB)
    bj = Jc * R * SB + w % (R * SB)
    return bi, bj, (bi < nbi and bj < nbj and bj < R * bi + R)


def n_slots(nbi, nbj, R):
    nJ = (nbj + R * SB - 1) // (R * SB)
    nI = (nbi + SB - 1) // SB
    nsb = nI * (nI + 1) // 2 if nI <= nJ else nJ * (nJ + 1) // 2 + (nI - nJ) * nJ
    return nsb * SB * R * SB


@pytest.mark.parametrize("n_tiles128", [1, 2, 7, 16, 17, 33, 64, 100])
def test_superblocked_enumeration_covers_lower_triangle_once(n_tiles128):
    for R in (2, 4):  # 64-column tiles (up to 4 slices) and 32-column tiles (5 and more)
        _check_superblocked(n_tiles128, R)


def _check_superblocked(n_tiles128, R):
    # the Cholesky shape: N = n_tiles128*128 columns, M = N + 128 border rows
    nbi, nbj = n_tiles128 + 1, R * n_tiles128
    want = {(bi, bj) for bi in range(nbi) for bj in range(min(nbj, R * bi + R))}  # BN-col tile bj below 128-row tile bi
    got = []
    for t in range(n_slots(nbi, nbj, R)):
        bi, bj, ok = oz_tile(t, nbi, nbj, R)
        if ok:
            got.append((bi, bj))
    assert len(got) == len(set(got)), "a tile is visited twice"
    assert set(got) == want


def strip_table(nbi, nbj, b_tile_stride, b_tile_width, b_off, a_off, BN):
    start, bimin, n = [], [], 0
    bw = b_tile_width or 128
    for j in range(nbj):
        n0 = j * BN
        nsrc = ((n0 // bw) * b_tile_stride + n0 % bw if b_tile_stride else n0) + b_off
        bm = (nsrc - a_off) // 128 if nsrc - a_off >= 0 else 0
        bm = min(bm, nbi)
        bimin.append(bm)
        start.append(n)
        n += nbi - bm
    start.append(n)
    return start, bimin, n


def tab_decode(t, start, bimin, nbj):
    lo, hi = 0, nbj
    while hi - lo > 1:
        mid = (lo + hi) >> 1
        if start[mid] <= t:
            lo = mid
        else:
            hi = mid
    return bimin[lo] + (t - start[lo]), lo


@pytest.mark.parametrize("R,me,W,kk,nto", [(2, 0, 256, 0, 7), (2, 1, 256, 1, 7), (4, 3, 512, 2, 16), (8, 5, 512, 0, 20), (3, 0, 128, 4, 11)])
def test_block_cyclic_strip_table(R, me, W, kk, nto):
    """rank `me` of R updates its local outer blocks with global index > kk after outer step kk; the rows of the
    packed panel start at global row (kk+1)*W; a local column tile must see exactly the row tiles at/below it"""
    local = [j for j in range(nto) if j % R == me and j > kk]
    if not local:
        pytest.skip("no local trailing blocks")
    for BN in (64, 32):  # strip width of the up-to-4-slice and of the longer splits
        _check_strip_table(R, W, kk, nto, local, BN)


def _check_strip_table(R, W, kk, nto, local, BN):
    rows_below = (nto - (kk + 1)) * W + 128
    nbi, nbj = (rows_below + 127) // 128, len(local) * W // BN
    b_off = (local[0] - (kk + 1)) * W
    start, bimin, n = strip_table(nbi, nbj, R * W, W, b_off, 0, BN)
    seen = set()
    for t in range(n):
        bi, bj = tab_decode(t, start, bimin, nbj)
        assert (bi, bj) not in seen
        seen.add((bi, bj))
    want = set()
    for bj in range(nbj):
        n0 = bj * BN
        jglob = local[n0 // W]                       # global outer block of this local column tile
        prow = (jglob - (kk + 1)) * W + n0 % W       # its row in the packed panel
        assert prow == (n0 // W) * R * W + n0 % W + b_off
        for bi in range(nbi):
            if prow < bi * 128 + 128:                # tile touches the lower triangle (incl. diagonal-crossing)
                want.add((bi, bj))
    assert seen == want
