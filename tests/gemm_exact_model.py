"""Exact model of the tile GEMM (csrc/gemm.cu) as the kernels run it, for agp_debug_gemm: which kernel a product selects
and its tile, the tiles lower_only skips, the block-cyclic column map, the K cut-off of trmm_lower and the owned set (every
entry of a computed tile, clipped to M x N).  Values are exact: the test data are integers scaled by per-row (A) and
per-column (B) powers of two, so every partial sum is a multiple of one unit and stays below 2^53 (fp64) or 2^24 (fp32)
units -- exact in any summation order.  The model asserts that condition for every owned entry, so an owned entry of the
kernel must equal the model bit for bit; everything else in the C buffer must be unchanged.

Buffers are flat NumPy arrays laid out as the device buffers: A(m, k) at A[m + k*lda] (a_kmajor = 0) or A[k + m*lda],
B(k, n) at B[n + k*ldb] (b_kmajor = 0) or B[k + n*ldb], C(m, n) at C[m + n*ldc].  In-place products pass the same array
object for C and the operand, as the library takes the same pointer."""
from dataclasses import dataclass, replace

import numpy as np


@dataclass(frozen=True)
class Gemm:
    dtype: type            # np.float64 | np.float32
    M: int
    N: int
    K: int
    a_kmajor: int = 0
    lda: int = 0
    b_kmajor: int = 0
    ldb: int = 0
    ldc: int = 0
    alpha_neg: int = 0
    beta_one: int = 0
    lower_only: int = 0
    trmm_lower: int = 0
    stride: int = 0        # b_tile_stride
    width: int = 0         # b_tile_width (0 -> 128)
    b_off: int = 0
    alias: str = ""        # "" | "A" (C == A) | "B" (C == B)
    a_misalign: int = 0    # element offsets of the pointers passed (contract tests only)
    b_misalign: int = 0
    c_misalign: int = 0


def vec(dtype):
    """elements per 16-byte load"""
    return 16 // np.dtype(dtype).itemsize


def tile(g):
    """(TBM, TBN) of the kernel the product selects"""
    if g.dtype == np.float32:
        return 128, 128
    return {"A": (64, 128), "B": (128, 128), "": (128, 64)}[g.alias]


def kernel_name(g):
    if g.dtype == np.float32:
        return "gemm_simt_kernel<%d,%d>" % (g.a_kmajor, g.b_kmajor)
    wm, wn = {"A": (1, 4), "B": (2, 4), "": (2, 2)}[g.alias]
    return "gemm_dmma_kernel<%d,%d,%d,%d>" % (g.a_kmajor, g.b_kmajor, wm, wn)


def col_source(g, n):
    """B column read by C column n (the block-cyclic map; identity without a stride)"""
    n = np.asarray(n, dtype=np.int64)
    if not g.stride:
        return n
    bw = g.width or 128
    return (n // bw) * g.stride + n % bw + g.b_off


def highest_b_column(g):
    if g.N <= 0:
        return -1
    return int(col_source(g, np.arange(g.N)).max())


def contract_ok(g):
    """mirror of gemm_contract_ok (csrc/gemm.cu) for a product with M, N > 0"""
    V = vec(g.dtype)
    if g.K < 0 or g.a_misalign % V or g.b_misalign % V or g.lda % V or g.ldb % V:
        return False
    if g.dtype == np.float32 and (g.c_misalign % V or g.ldc % V or g.M % V):
        return False
    if (g.a_kmajor or g.b_kmajor) and g.K % V:
        return False
    if g.stride:
        bw = g.width or 128
        if g.stride < 0 or g.width < 0 or g.b_off < 0 or bw % tile(g)[1]:
            return False
        if not g.b_kmajor and ((g.stride - bw) % V or g.b_off % V):
            return False
    if g.lda < (g.K if g.a_kmajor else g.M) or g.ldb < (g.K if g.b_kmajor else highest_b_column(g) + 1) or g.ldc < g.M:
        return False
    if g.alias == "A" and (g.a_kmajor or g.ldc != g.lda or g.N > 128):
        return False
    if g.alias == "B" and (not g.b_kmajor or g.ldc != g.ldb or g.M > 128 or g.stride):
        return False
    return True


def owned(g, tbm=None, tbn=None):
    """M x N mask of the entries the kernel writes, and the K each row reads (trmm_lower cuts it per row tile)"""
    TBM, TBN = tile(g)
    TBM, TBN = tbm or TBM, tbn or TBN
    own = np.zeros((g.M, g.N), bool)
    for m0 in range(0, g.M, TBM):
        for n0 in range(0, g.N, TBN):
            if g.lower_only and int(col_source(g, n0)) >= m0 + TBM:
                continue
            own[m0:m0 + TBM, n0:n0 + TBN] = True
    kcut = np.full(g.M, g.K, dtype=np.int64)
    if g.trmm_lower:
        kcut = np.minimum(g.K, (np.arange(g.M) // TBM) * TBM + TBM)
    return own, kcut


def op_a(g, A):
    m, k = np.arange(g.M)[:, None], np.arange(g.K)[None, :]
    idx = (k + m * g.lda) if g.a_kmajor else (m + k * g.lda)
    return A[idx] if g.K else np.zeros((g.M, 0), A.dtype)


def op_b(g, B):
    k, n = np.arange(g.K)[:, None], col_source(g, np.arange(g.N))[None, :]
    idx = (k + n * g.ldb) if g.b_kmajor else (n + k * g.ldb)
    return B[idx] if g.K else np.zeros((0, g.N), B.dtype)


def c_index(g):
    return np.arange(g.M)[:, None] + np.arange(g.N)[None, :] * g.ldc


def low_exponent(x):
    """exponent of the lowest set bit of each |x| (+inf for 0): x is an integer multiple of 2^low_exponent(x)"""
    x = np.asarray(x, dtype=np.float64)
    f, e = np.frexp(np.abs(x))
    q = (f * 2.0 ** 53).astype(np.int64)
    tz = np.zeros(q.shape, np.int64)
    nz = q != 0
    qq = q[nz]
    tz[nz] = np.log2((qq & -qq).astype(np.float64)).astype(np.int64)
    out = (e - 53 + tz).astype(np.float64)
    out[~nz] = np.inf
    return out


def expected(g, A, B, Cbuf, tbm=None, tbn=None):
    """(C buffer after the call, owned mask).  A / B / Cbuf are the flat buffers before the call (the same object where
    C aliases an operand); the pointers passed are their starts."""
    want = Cbuf.copy()
    if g.M <= 0 or g.N <= 0:
        return want, np.zeros((max(g.M, 0), max(g.N, 0)), bool)
    own, kcut = owned(g, tbm, tbn)
    a = op_a(g, A).astype(np.float64)
    b = op_b(g, B).astype(np.float64)
    ci = c_index(g)
    c = Cbuf[ci].astype(np.float64) if g.beta_one else np.zeros((g.M, g.N))
    acc = np.zeros((g.M, g.N))
    bound = np.abs(c).copy()
    for kc in np.unique(kcut):
        rows = kcut == kc
        acc[rows] = a[rows, :kc] @ b[:kc]
        bound[rows] += np.abs(a[rows, :kc]) @ np.abs(b[:kc])
    # exactness: every term and c are integer multiples of 2^u, and the sum of their magnitudes is below 2^p units
    p = 53 if g.dtype == np.float64 else 24
    ua = low_exponent(a).min(axis=1, initial=np.inf)
    ub = low_exponent(b).min(axis=0, initial=np.inf)
    u = np.minimum(ua[:, None] + ub[None, :], low_exponent(c))
    u = np.where(np.isinf(u), 0.0, u)
    assert np.all(~own | (bound < np.ldexp(1.0, (p + u).astype(np.int64)))), "test data not exact in %d bits" % p
    with np.errstate(invalid="ignore"):
        val = (c - acc if g.alpha_neg else c + acc).astype(g.dtype)
    if g.dtype == np.float32 and g.alpha_neg and not g.beta_one:
        val = np.where(val == 0, np.float32(-0.0), val)  # the fp32 epilogue negates the sum: -(+0) = -0
    else:
        val = np.where(val == 0, g.dtype(0.0), val)      # fma(sign, acc, c) and x + (-x) round to +0
    want[ci[own]] = val[own]
    return want, own


# ---- test data ------------------------------------------------------------------------------------------------------------
def data_ranges(g):
    """integer bits and exponent ranges of A rows, B columns and C entries that keep g exact (see expected())"""
    if g.dtype == np.float64:
        bits, ra, cb = 13, (-16, 16), (-16, 16)
    else:
        bits, ra, cb = 5, (-8, 8), (-8, 8)
    if g.alias == "A":   # C holds A's values (unit 2^ra): column scales at most 1
        cb = (cb[0], 0)
    if g.alias == "B":   # C holds B's values (unit 2^cb): row scales at most 1
        ra = (ra[0], 0)
    return bits, ra, cb


def make_buffers(g, rng, pad_value=np.nan, tail=37):
    """flat A, B, C buffers for g: op(A), the B columns the map reads and C hold scaled integers; every other element (ld
    padding, B columns the map skips, a tail past each buffer) holds pad_value.  Aliased products return the same array
    for C and the operand, sized for both roles."""
    bits, ra, cb = data_ranges(g)
    M, N, K, dt = g.M, g.N, g.K, g.dtype
    ncol_b = highest_b_column(g) + 1
    erow = rng.integers(ra[0], ra[1] + 1, M)
    ecol = rng.integers(cb[0], cb[1] + 1, max(ncol_b, N))

    def ints(shape):
        return (rng.integers(1, 2 ** bits + 1, shape) * rng.choice([-1, 1], shape)).astype(np.float64)

    def fill(ld, ncols, rows_idx, cols_idx, kmajor, vals):
        buf = np.full(ld * ncols + tail, pad_value, dtype=dt)
        r, c = np.asarray(rows_idx)[:, None], np.asarray(cols_idx)[None, :]
        if vals.size:
            buf[(c + r * ld) if kmajor else (r + c * ld)] = vals.astype(dt)
        return buf

    # A: M x KA (C == A also keeps C's N columns there); element (m, k) stored at [m + k*lda] or [k + m*lda]
    KA = max(K, N) if g.alias == "A" else K
    A = fill(g.lda, KA if not g.a_kmajor else M, range(M), range(KA), g.a_kmajor, ints((M, KA)) * np.ldexp(1.0, erow)[:, None])
    # B: KB x (the columns the map reads); element (k, n) at [n + k*ldb] or [k + n*ldb] (fill's rows = n, cols = k)
    KB = max(K, M) if g.alias == "B" else K
    cols = np.arange(N) if g.alias == "B" else np.unique(col_source(g, np.arange(N)))
    bv = ints((KB, cols.size)) * np.ldexp(1.0, ecol[cols])[None, :]
    B = fill(g.ldb, ncol_b if g.b_kmajor else KB, cols, range(KB), g.b_kmajor, bv.T)
    if g.alias == "A":
        return A, B, A
    if g.alias == "B":
        return A, B, B
    Cbuf = np.full(g.ldc * N + tail, pad_value, dtype=dt)
    Cbuf[c_index(g)] = (ints((M, N)) * np.ldexp(1.0, erow[:, None] + ecol[col_source(g, np.arange(N))][None, :]) * 0.5).astype(dt)
    return A, B, Cbuf


def with_lds(g, extra=0):
    """g with the smallest aligned leading dimensions for its storage (plus `extra` aligned elements of padding)"""
    V = vec(g.dtype)
    up = lambda x: max(V, -(-x // V) * V) + extra * V
    rows_a = g.K if g.a_kmajor else g.M
    rows_b = g.K if g.b_kmajor else highest_b_column(g) + 1
    if g.alias == "A":
        lda = up(g.M)
        return replace(g, lda=lda, ldc=lda, ldb=up(rows_b))
    if g.alias == "B":
        ldb = up(max(g.K, g.M))
        return replace(g, ldb=ldb, ldc=ldb, lda=up(rows_a))
    return replace(g, lda=up(rows_a), ldb=up(rows_b), ldc=up(g.M))


# ---- the cases the device test runs ------------------------------------------------------------------------------------
MN = [1, 4, 63, 64, 65, 128, 129, 300]
KS = [0, 2, 4, 16, 18, 48, 130, 1030]
# every kernel the product can select under the contract: C == A needs A MN-major, C == B needs B K-major
INSTANTIATIONS = [(dt, akm, bkm, alias) for dt in (np.float64, np.float32)
                  for alias, layouts in (("", [(0, 0), (0, 1), (1, 0), (1, 1)]), ("A", [(0, 0), (0, 1)]), ("B", [(0, 1), (1, 1)]))
                  for akm, bkm in layouts]


def instantiation_cases(dt, akm, bkm, alias):
    """(M, N, K) x flags for one kernel: every M, N and K of MN / KS that the contract allows (fp32: M % 4 == 0, K % 4 ==
    0 with a K-major operand, N > 1; C == A: N <= 128; C == B: M <= 128), cycled against each other so each value meets
    several partners, each with alpha = +-1 x beta in {0, 1} and alternately lower_only / trmm_lower, ld padding 0 or 1"""
    V = vec(dt)
    Ms = [m for m in MN if (dt == np.float64 or m % V == 0) and (alias != "B" or m <= 128)]
    Ns = [n for n in MN if (dt == np.float64 or n > 1) and (alias != "A" or n <= 128)]
    Ks = [k for k in KS if not (akm or bkm) or k % V == 0]
    if dt == np.float32 and (akm or bkm):
        Ks += [132, 1028]
    count = max(len(Ms), len(Ns), len(Ks))
    out = []
    for i in range(count):
        M, N, K = Ms[i % len(Ms)], Ns[(i + 3) % len(Ns)], Ks[(i + 5) % len(Ks)]
        for j, (an, b1) in enumerate([(0, 0), (1, 1), (1, 0), (0, 1)]):
            flags = dict(alpha_neg=an, beta_one=b1, lower_only=int((i + j) % 3 == 1), trmm_lower=int((i + j) % 3 == 2))
            g = Gemm(dt, M, N, K, a_kmajor=akm, b_kmajor=bkm, alias=alias, **flags)
            out.append(with_lds(g, extra=(i + j) % 2))
    return out


def pinning_cases(dt, akm, bkm, alias):
    """products whose owned set or K cut-off depends on the tile: lower_only and trmm_lower over several row tiles, and
    for separate operands lower_only through a map that shifts columns by 64, where 64- and 128-wide column tiles differ"""
    M = 128 if alias == "B" else 300
    N = 128 if alias == "A" else 300
    flags = [dict(lower_only=1), dict(trmm_lower=1)]
    if alias == "":
        flags.append(dict(lower_only=1, stride=128, b_off=64))
    return [with_lds(Gemm(dt, M, N, 256, a_kmajor=akm, b_kmajor=bkm, alias=alias, alpha_neg=1, beta_one=1, **f))
            for f in flags]


def other_tiles(g):
    """the tiles of the fp64 kernels g did not select whose output on the pinning products differs from g's: C == B's
    128 x 128 tile and the separate kernel's 128 x 64 one own the same entries unless a map shifts the columns, which
    the in-place kernel refuses, so between those two only the separate products are pinned"""
    if g.dtype == np.float32:
        return []
    return {"": [(64, 128), (128, 128)], "A": [(128, 64), (128, 128)], "B": [(64, 128)]}[g.alias]


# the column maps fit_dist_impl builds: R ranks x blocks of W columns, local column n of rank `me` reads panel row
# (n / W) * R * W + n % W + b_off (b_off = the rank's first block, minus the panel's first row)
def map_cases(dt):
    out = []
    for R, W, offs in ((2, 128, (0, 128)), (4, 128, (256, 384)), (8, 128, (896,)), (2, 512, (0, 512)), (4, 512, (1024,))):
        for b_off in offs:
            N = 2 * W + (128 if W == 128 else 256)
            M = (N // W) * R * W + b_off  # rows of the panel below the diagonal block: reaches the last column read
            M = min(M, 1200)
            for bkm, lo in ((0, 1), (1, 1), (0, 0)):
                g = Gemm(dt, M, N, 128, a_kmajor=0, b_kmajor=bkm, alpha_neg=1, beta_one=1, lower_only=lo, stride=R * W,
                         width=W, b_off=b_off)
                out.append(with_lds(g))
    return out
