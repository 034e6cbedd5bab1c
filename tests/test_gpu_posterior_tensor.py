"""The exact posterior's follow-on operations at the sizes where they run on the tensor cores, against the fp64 oracle
(oracle/agp_ref.py) and LAPACK's dpotrf for the expected pivots:

  operation (engine.cu)                                 tensor-core branch                  cases
  post_extend_impl: Cholesky of C22 - L21 L21'          int8-slice trailing update,         test_extend_forced_fp64,
    (cholesky_inplace with lda != rows_total, the         512-wide panels                     test_extend_auto_fp64,
    sub-matrix at row / column n1_pad)                                                        test_extend_auto_fp32,
                                                                                              test_not_posdef_extension_on_int8_panels
  post_cond_impl: Cholesky of K** + S* - V'V            same                                test_post_cond,
    (logpdf / rand of a FiniteGP over the posterior)                                          test_extend_forced_fp64 (over an extended
                                                                                              handle), test_extend_auto_fp64 (chain
                                                                                              rule), test_not_posdef_post_cond_on_int8_panels
  forward_subst_multi in post_cond / post_mean_cov /    two-level substitution, int8        every case; over a factor with padded gap
    post_solve_lower / post_mean_var                      rank-512 updates                    rows: test_extend_*; plain handle:
                                                                                              test_plain_handle_mean_cov_and_solves
  ctx->oz re-used across calls of other sizes           --                                  test_slice_workspace_reuse_across_sizes

Which branch ran is asserted from the launch counter: the same call runs under the tensor policy and under tensor mode 0
with the same tile_nb, and the difference is compared with a model of the launches (`_chol_trailing`, and
`_subst_launches` of tests/test_gpu_vfe_tensor.py).  Each case also asserts that an output without fp64 atomics (alpha,
the variances, the solves, the rand draws) has different bits in the two modes.

Data: C2-like for fp64 (SqExponential, ScaleTransform, 8 features, noise 0.1), C3-like for fp32 (Matern-3/2, ARD over 8
features, noise 0.05); per-point noise in [0.05, 0.1] on the new points of every extension.

Tolerances.  fp64: logpdf / logdet rtol 1e-8 (BASELINE.json); alpha rtol 1e-6 with atol 1e-7 max|alpha|; U, means,
variances, covariances and solves element-wise at 1e-7.  fp32 (`_Tol32`): logdet rtol 1e-4, logpdf over the posterior
1e-4 of its terms (M log(2 pi) / 2 + |logpdf|), element-wise bounds from the conditioning of C = K + S = L L'
(derivation in `_Tol32`)."""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import lapack

from oracle import agp_ref as ref
from test_gpu_vfe_tensor import _subst_launches

pytestmark = pytest.mark.gpu

TILE = 128
EPS32 = float(np.finfo(np.float32).eps)
FORCED = dict(fp64_mode=1, fp32_mode=-1, tile_nb=512)      # below the automatic thresholds: int8 slices, 512-wide panels
FORCED_OFF = dict(fp64_mode=0, fp32_mode=-1, tile_nb=512)  # the same panels on the DMMA kernels
AUTO = dict(fp64_mode=-1, fp32_mode=-1, tile_nb=0)
AUTO_OFF = dict(fp64_mode=0, fp32_mode=0, tile_nb=0)


def _rup(x, m=TILE):
    return (x + m - 1) // m * m


@pytest.fixture
def eng(ag):
    """the engine under the automatic policy; whatever a case sets is put back"""
    e = ag.engine()
    c = e.get_config()
    old = (c.fp64_mode, c.fp32_mode, c.tile_nb)
    assert old == (-1, -1, 0), "automatic policy expected"
    assert c.lookahead == 2, "the launch model below is written for the default look-ahead"
    try:
        yield e
    finally:
        e.set_config(fp64_mode=old[0], fp32_mode=old[1], tile_nb=old[2])


def _chol_trailing(n_pad, G, int8):
    """(launches, int8 panels) of the trailing updates of cholesky_inplace at look-ahead 2 (the panel factorisations are
    the same in both modes and left out).  An outer panel of G blocks takes the int8 path when it is full width (K = 512
    = the workspace's K), at least 256 columns trail it and nblk > 2G: the slices are prepared (row scales + slices, two
    launches), then the next panel and the rest are updated by one int8 launch each.  Every other panel takes the depth-2
    look-ahead branch of the tile GEMM: the next panel, then the rest split into the panel after next (restA) and the
    remainder (restB), one launch each.  So an int8 panel adds two launches over the GEMM schedule, less one when the
    GEMM schedule has a restB."""
    nblk = n_pad // TILE
    la = nblk > 2 * G
    total = panels = 0
    for ko in range(0, nblk, G):
        g_end = min(ko + G, nblk)
        t0 = g_end * TILE
        cols_trail = n_pad - t0
        if cols_trail <= 0:
            continue
        nxt = min(cols_trail, G * TILE)
        if int8 and la and g_end - ko == G and cols_trail >= 2 * TILE:
            total += 2 + 1 + (cols_trail > nxt)
            panels += 1
        elif not la:
            total += 1
        else:
            total += 1
            if cols_trail > nxt:
                r0 = t0 + nxt
                total += 1 + (n_pad > r0 + min(n_pad - r0, G * TILE))
    return total, panels


def _chol_delta(n_pad, G=4):
    """launches the int8-slice Cholesky adds over tensor mode 0 at the same panel width, and its number of int8 panels"""
    on, panels = _chol_trailing(n_pad, G, True)
    return on - _chol_trailing(n_pad, G, False)[0], panels


def _subst_delta(n_pad, ncols):
    return _subst_launches(n_pad, ncols, True) - _subst_launches(n_pad, ncols, False)


def _on_off(eng, on, off, call):
    """(result, launches) of call() under the config `on`, then under `off`; `on` is left set"""
    out = []
    for cfg in (off, on):
        eng.set_config(**cfg)
        l0 = eng.launch_count()
        r = call()
        out.append((r, eng.launch_count() - l0))
    return out[1] + out[0]


class Data:
    """C2-like (fp64) or C3-like (fp32) points; the oracle sees the fp64 image of the same bytes"""

    def __init__(self, ag, dtype, n, mean_c=0.0, d=8):
        self.ag, self.dtype = ag, dtype
        if dtype == np.float64:
            cfg = ref.make_config("C2", n=n)
            self.X, self.s2 = np.ascontiguousarray(cfg["X"][:, :d]), 0.1
            self.ks = ref.KernelSpec(ref.SE, 1.0, ref.T_SCALE, scale=1.0 / (0.5 * np.sqrt(d)))
            kern = ag.SqExponentialKernel().compose(ag.ScaleTransform(self.ks.scale))
        else:
            cfg = ref.make_config("C3", n=n)
            self.X, self.s2 = np.ascontiguousarray(cfg["X"][:, :d]), 0.05
            ard = np.ascontiguousarray(cfg["k"].ard[:d]) * np.float32(np.sqrt(32.0 / d))
            self.ks = ref.KernelSpec(ref.MATERN32, 1.0, ref.T_ARD, ard=ard.astype(np.float64))
            kern = ag.Matern32Kernel().compose(ag.ARDTransform(ard))
        self.y = cfg["y"]
        rng = np.random.default_rng(n)
        self.nv = (0.05 + 0.05 * rng.random(n)).astype(dtype)  # per-point noise of the extensions
        self.Xs = rng.random((1536, d)).astype(dtype)
        self.mean_c = mean_c
        self.f = ag.GP(mean_c, kern) if mean_c else ag.GP(kern)
        self.mean = ref.MeanSpec(1, mean_c) if mean_c else ref.MeanSpec()

    def seg(self, a, b):
        return self.X[a:b], self.y[a:b]

    def oracle(self, n, noise):
        """ref.posterior over the first n points with the noise vector `noise` (fp64)"""
        return ref.posterior(self.ks, self.mean, ref.NoiseSpec(1, v=np.asarray(noise, np.float64)),
                             self.X[:n].astype(np.float64), self.y[:n].astype(np.float64))


def _lam_max(U, its=40):
    """largest eigenvalue of U'U by power iteration"""
    x = np.random.default_rng(0).standard_normal(U.shape[0])
    lam = 0.0
    for _ in range(its):
        w = U.T @ (U @ x)
        lam = float(np.linalg.norm(w) / np.linalg.norm(x))
        x = w / np.linalg.norm(w)
    return lam


class _Tol64:
    lp = 1e-8

    def __init__(self, pr, noise_min):
        pass

    def alpha(self, a):
        return dict(rtol=1e-6, atol=1e-7 * float(np.abs(a).max()))

    mean = var = U = dict(rtol=1e-6, atol=1e-7)
    rand = dict(rtol=0, atol=1e-7)


class _Tol32:
    """fp32 element-wise bounds from cond = cond(C), C = K + S = L L' (lambda_min >= min noise, lambda_max by power
    iteration on the oracle's factor).  The factorisation and the substitutions are backward stable: the computed
    a = L^-1 k solves (L + dL) a = k with |dL| <= g eps32 |L|, so |da| / |a| <= g eps32 sqrt(cond).  Each column a of
    V = L^-1 K(x, x*) has |a|^2 <= k(x*, x*) = 1, so V, V'V, a variance k** - |a|^2 and a covariance carry at most
    2 g eps32 sqrt(cond).  A mean is a' v with v = L^-1 delta: 2 g eps32 sqrt(cond) |v|.  alpha = L'^-1 v loses
    g eps32 cond relative to max|alpha|, and so does U (the forward error of a Cholesky factor).  g = 4 is held here;
    the worst case is n eps32, rounding errors of both signs leave far less (measured figures in DESIGN.md s6)."""
    lp = 1e-4

    def __init__(self, pr, noise_min):
        self.cond = _lam_max(pr["U"]) / noise_min
        sq = 8 * EPS32 * np.sqrt(self.cond)
        vnorm = float(np.sqrt(max(pr["delta"] @ pr["alpha"], 1.0)))
        self.mean = dict(rtol=0, atol=sq * vnorm)
        self.var = dict(rtol=0, atol=sq)
        self.U = dict(rtol=0, atol=4 * EPS32 * self.cond * float(np.abs(pr["U"]).max()))
        self.rand = dict(rtol=0, atol=self.mean["atol"] + 4 * sq / np.sqrt(noise_min))

    def alpha(self, a):
        return dict(rtol=0, atol=4 * EPS32 * self.cond * float(np.abs(a).max()))


def _tol(dtype, pr, noise_min):
    return (_Tol64 if dtype == np.float64 else _Tol32)(pr, noise_min)


def _err(got, want):
    return float(np.abs(np.asarray(got, np.float64) - want).max())


def _rel(got, want):
    return abs(float(got) - want) / abs(want)


def _check_predictions(ag, eng, post, pr, data, n_pad, on, off, tol, n_cov=640, tag=""):
    """mean_and_var at 1536 points (launches and bits under both modes), mean_and_cov at the first n_cov, solve_lower /
    Xt_invA_X with 512 (tensor substitution) and 130 (tile path) columns, Xt_invA_Y, diag_Xt_invA_X and tr_Xt_invA_X
    with 512.  One oracle solve V = U'^-1 K(x, x*) serves all of them; the right-hand sides are columns of K(x, x*)."""
    Xs, Xs64 = data.Xs, data.Xs.astype(np.float64)
    Kxs = ref.kernelmatrix(pr["k"], pr["x"], Xs64)
    V = ref._Ut_solve(pr["U"], Kxs)
    mu_r = pr["mean"].vector(len(Xs), np.float64) + Kxs.T @ pr["alpha"]
    v_r = ref.kernelmatrix_diag(pr["k"], Xs64) - np.sum(V * V, 0)
    (mu, v), l_on, (mu0, v0), l_off = _on_off(eng, on, off, lambda: ag.mean_and_var(post, ag.RowVecs(Xs)))
    assert l_on - l_off == _subst_delta(n_pad, 1536) != 0, (l_on, l_off)
    assert not np.array_equal(v, v0)
    print(tag, "mean_and_var", _err(mu, mu_r), _err(v, v_r), _err(v0, v_r))
    assert np.allclose(mu, mu_r, **tol.mean) and np.allclose(v, v_r, **tol.var), (_err(mu, mu_r), _err(v, v_r))
    assert np.allclose(mu0, mu_r, **tol.mean) and np.allclose(v0, v_r, **tol.var)

    mc, Cc = ag.mean_and_cov(post, ag.RowVecs(Xs[:n_cov]))
    Cr = ref.kernelmatrix(pr["k"], Xs64[:n_cov]) - V[:, :n_cov].T @ V[:, :n_cov]
    print(tag, "mean_and_cov", _err(mc, mu_r[:n_cov]), _err(Cc, Cr), _err(Cc, Cc.T))
    assert np.allclose(mc, mu_r[:n_cov], **tol.mean) and np.allclose(Cc, Cr, **tol.var), _err(Cc, Cr)
    # V'V: entry (i, j) and (j, i) are dot products of the same columns: n_pad roundings of size <= eps k(x*, x*)
    assert _err(Cc, Cc.T) <= n_pad * np.finfo(data.dtype).eps, _err(Cc, Cc.T)

    A = post.data.C
    B = np.asfortranarray(Kxs[:, :1024].astype(data.dtype))
    V512, l_on, V512_0, l_off = _on_off(eng, on, off, lambda: A.solve_lower(B[:, :512]))
    assert l_on - l_off == _subst_delta(n_pad, 512) != 0, (l_on, l_off)
    assert not np.array_equal(V512, V512_0)
    V130 = A.solve_lower(B[:, :130])
    print(tag, "solve_lower", _err(V512, V[:, :512]), _err(V130, V512[:, :130]))
    assert np.allclose(V512, V[:, :512], **tol.var) and np.allclose(V130, V[:, :130], **tol.var)
    # the tile path and the tensor path: each within the oracle's bound, hence within twice that of each other
    assert np.allclose(V130, V512[:, :130], rtol=0, atol=2 * tol.var["atol"])
    G = V[:, :512].T @ V[:, :512]
    assert np.allclose(ag.Xt_invA_X(A, B[:, :512]), G, **tol.var)
    assert np.allclose(ag.Xt_invA_X(A, B[:, :130]), G[:130, :130], **tol.var)
    assert np.allclose(ag.Xt_invA_Y(B[:, :512], A, B[:, 512:]), V[:, :512].T @ V[:, 512:1024], **tol.var)
    assert np.allclose(ag.diag_Xt_invA_X(A, B[:, :512]), np.diag(G), **tol.var)
    assert _rel(ag.tr_Xt_invA_X(A, B[:, :512]), np.trace(G)) <= (1e-8 if data.dtype == np.float64 else 1e-4)


def _check_handle(post, pr, n, tol, export, tag=""):
    a = post.data.alpha
    print(tag, "alpha", _err(a, pr["alpha"]) / np.abs(pr["alpha"]).max(), "logdet",
          _rel(post.data.C.logdet(), ref.logdet_chol(pr["U"])))
    assert post.data.C.n == n
    assert np.allclose(a, pr["alpha"], **tol.alpha(pr["alpha"])), _err(a, pr["alpha"])
    assert np.allclose(post.data.delta, pr["delta"], rtol=0, atol=4 * np.finfo(a.dtype).eps * np.abs(pr["delta"]).max())
    assert _rel(post.data.C.logdet(), ref.logdet_chol(pr["U"])) <= tol.lp
    if export:
        U = post.data.C.U
        print(tag, "U", _err(U, pr["U"]))
        assert np.allclose(U, pr["U"], **tol.U), _err(U, pr["U"])


def _cond_oracle(pr, Xs, noise_s):
    """mean and upper factor of the posterior covariance at Xs plus noise_s: ref.post_logpdf and ref.post_rand_from_Z
    up to their last step, computed once for both"""
    m, Cs = ref.post_mean_and_cov(pr, Xs)
    Cs[np.diag_indices(len(Xs))] += noise_s
    return m, ref.cholesky_upper(Cs)


def _check_post_cond(ag, eng, post, pr, data, Xs, n_pad, on, off, tol, G=4, tag=""):
    """logpdf of a FiniteGP over the posterior with 3 and 130 columns (two calls of the 128-column C ABI), rand with 4"""
    M, dt, s2 = len(Xs), data.dtype, data.s2
    m, Us = _cond_oracle(pr, Xs.astype(np.float64), s2)
    rng = np.random.default_rng(M)
    Y = (m[:, None] + Us.T @ rng.standard_normal((M, 130))).astype(dt)
    r = Y.astype(np.float64) - m[:, None]
    want = -0.5 * (M * ref.LOG2PI + ref.logdet_chol(Us) + ref.diag_Xt_invA_X(Us, r))
    fx = post(ag.RowVecs(Xs), s2)
    lp, l_on, lp0, l_off = _on_off(eng, on, off, lambda: ag.logpdf(fx, np.asfortranarray(Y[:, :3])))
    m_pad = _rup(M)
    if dt == np.float64:
        dc, panels = _chol_delta(m_pad, G)
        assert panels > 0 and l_on - l_off == _subst_delta(n_pad, m_pad) + dc, (l_on, l_off, dc)
    else:
        assert l_on != l_off, l_on
    lp130 = ag.logpdf(fx, Y)
    # fp64: rtol 1e-8 of the value.  fp32: the value is a small difference of terms of size M log(2 pi) / 2 (logdet and
    # the quadratic form are each of order M): rounding hits the terms, so 1e-4 is held of the terms, not of the rest
    # (as for the VFE posterior in test_gpu_vfe_tensor.py)
    scale = np.abs(want) if dt == np.float64 else 0.5 * M * ref.LOG2PI + np.abs(want)
    lp_tol = tol.lp
    print(tag, "post_cond logpdf", M, np.max(np.abs(lp - want[:3]) / np.abs(want[:3])),
          np.max(np.abs(lp130 - want) / np.abs(want)), np.max(np.abs(lp0 - want[:3]) / np.abs(want[:3])),
          np.max(np.abs(lp130 - want) / scale))
    assert np.all(np.abs(lp - want[:3]) <= lp_tol * scale[:3]), (lp, want[:3])
    assert np.all(np.abs(lp0 - want[:3]) <= lp_tol * scale[:3]), (lp0, want[:3])
    assert np.all(np.abs(lp130 - want) <= lp_tol * scale), np.max(np.abs(lp130 - want) / scale)
    Z = np.asfortranarray(rng.standard_normal((M, 4)).astype(dt))
    want_r = m[:, None] + Us.T @ Z.astype(np.float64)
    got, _, got0, _ = _on_off(eng, on, off, lambda: ag.rand_from_normals(fx, Z))
    assert not np.array_equal(got, got0)
    if dt == np.float64:
        atol = 1e-7 * max(1.0, float(np.abs(want_r).max()))
    else:  # the mean's bound of _Tol32, plus U*' Z with U* the factor of C* + S*: 2 g eps32 sqrt(cond(C* + S*)) relative
        atol = tol.mean["atol"] + 8 * EPS32 * np.sqrt(_lam_max(Us) / s2) * float(np.abs(want_r - m[:, None]).max())
    print(tag, "post_cond rand", M, _err(got, want_r), _err(got0, want_r), atol)
    assert np.allclose(got, want_r, rtol=0, atol=atol) and np.allclose(got0, want_r, rtol=0, atol=atol)


# ---- A: sequential conditioning on the int8-slice Schur Cholesky ------------------------------------------------------
def _extend(ag, eng, data, n1, n2, on, off):
    """p1 on the first n1 points (scalar noise), p2 = posterior(p1(x2, s2), y2) with per-point noise, under both modes;
    returns p1, p2 (tensor mode), the oracle noise vector and the launch counts"""
    X1, y1 = data.seg(0, n1)
    X2, y2 = data.seg(n1, n1 + n2)
    eng.set_config(**on)
    p1 = ag.posterior(data.f(ag.RowVecs(X1), data.s2), y1)
    before = ag.mean_and_var(p1, ag.RowVecs(data.Xs[:300]))
    s2v = data.nv[n1:n1 + n2]
    p2, l_on, p2_0, l_off = _on_off(eng, on, off, lambda: ag.posterior(p1(ag.RowVecs(X2), s2v), y2))
    assert not np.array_equal(p2.data.alpha, p2_0.data.alpha)
    after = ag.mean_and_var(p1, ag.RowVecs(data.Xs[:300]))
    # value semantics: the handle conditioned on answers bit for bit as before
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    noise = np.concatenate([np.full(n1, data.s2), s2v.astype(np.float64)])
    return p1, p2, p2_0, noise, l_on, l_off


@pytest.mark.parametrize("n2", [1300, 2304])
def test_extend_forced_fp64(ag, eng, n2):
    """n1 = 700 (n1_pad = 768: 68 identity rows in the middle of the extended factor), constant mean 0.3, the new points
    with per-point noise; the Schur Cholesky of n2_pad x n2_pad on forced int8 panels.  n2 = 1300 also carries a third
    extension of 300 points (two gaps), the in-place extension of a second handle, and logpdf / rand at M = 1300 over the
    extended handle (the gapped substitution and the M x M int8 Cholesky in one call)."""
    n1 = 700
    data = Data(ag, np.float64, n1 + n2 + 300, mean_c=0.3)
    Xs = data.Xs
    p1, p2, p2_0, noise, l_on, l_off = _extend(ag, eng, data, n1, n2, FORCED, FORCED_OFF)
    dc, panels = _chol_delta(_rup(n2))
    assert panels == {1300: 2, 2304: 4}[n2] and l_on - l_off == dc, (l_on, l_off, dc)
    n, n_pad = n1 + n2, _rup(n1) + _rup(n2)
    pr = data.oracle(n, noise)
    tol = _Tol64(pr, 0.05)
    _check_handle(p2, pr, n, tol, export=True, tag="A forced %d" % n2)
    _check_handle(p2_0, pr, n, tol, export=False)
    _check_predictions(ag, eng, p2, pr, data, n_pad, FORCED, FORCED_OFF, tol, tag="A forced %d" % n2)
    if n2 != 1300:
        return
    _check_post_cond(ag, eng, p2, pr, data, Xs[:1300].copy(), n_pad, FORCED, FORCED_OFF, tol, tag="B over extended")

    # a third extension: the old factor now has two gaps (rows 700..767 and 2068..2175)
    X3, y3 = data.seg(n, n + 300)
    s3 = data.nv[n:n + 300]
    p3 = ag.posterior(p2(ag.RowVecs(X3), s3), y3)
    pr3 = data.oracle(n + 300, np.concatenate([noise, s3.astype(np.float64)]))
    _check_handle(p3, pr3, n + 300, tol, export=True, tag="A third")
    mu3, v3 = ag.mean_and_var(p3, ag.RowVecs(Xs))
    mu3r, v3r = ref.post_mean_and_var(pr3, Xs)
    print("A third mean_and_var", _err(mu3, mu3r), _err(v3, v3r))
    assert np.allclose(mu3, mu3r, **tol.mean) and np.allclose(v3, v3r, **tol.var)

    # in place: agp_post_extend with post_out = NULL on a second handle gives the same alpha bits
    api, cabi = ag.api, ag._cabi
    q = ag.posterior(data.f(ag.RowVecs(data.X[:n1]), data.s2), data.y[:n1])
    pts = api._Points(ag.RowVecs(data.X[n1:n])).astype(np.float64)
    keep = []
    ms = api._mean_struct(data.f.mean.spec(pts, np.float64), keep)
    ns = api._noise_struct(data.nv[n1:n], n2, np.float64, keep)
    y2 = np.ascontiguousarray(data.y[n1:n])
    alpha = np.empty(n, dtype=np.float64)
    eng.check(eng.L.agp_post_extend(q.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), n2, cabi.ptr(y2), C.byref(ms),
                                    C.byref(ns), cabi.ptr(alpha), None))
    assert q.data.C.n == n and np.array_equal(alpha, p2.data.alpha)
    assert q.data.C.logdet() == p2.data.C.logdet()


def test_extend_auto_fp64(ag, eng):
    """automatic policy: n1 = 1000, n2 = 8200 (n2_pad = 8320: int8 panels, then a 128-wide DMMA tail).  The U export is
    skipped (~9200^2 on the host).  The chain rule logpdf(fx1, y1) + logpdf(p1(x2, s2), y2) = logpdf(fx, y) runs the
    M x M Cholesky of post_cond at M = 8200 on the int8 path too."""
    n1, n2 = 1000, 8200
    data = Data(ag, np.float64, n1 + n2)
    p1, p2, p2_0, noise, l_on, l_off = _extend(ag, eng, data, n1, n2, AUTO, AUTO_OFF)
    dc, panels = _chol_delta(8320)
    assert panels == 15 and l_on - l_off == dc, (l_on, l_off, dc)
    del p2_0
    n, n_pad = n1 + n2, 1024 + 8320
    pr = data.oracle(n, noise)
    tol = _Tol64(pr, 0.05)
    _check_handle(p2, pr, n, tol, export=False, tag="A auto fp64")
    _check_predictions(ag, eng, p2, pr, data, n_pad, AUTO, AUTO_OFF, tol, tag="A auto fp64")
    del p2

    X1, y1 = data.seg(0, n1)
    X2, y2 = data.seg(n1, n)
    s2v = data.nv[n1:n]
    lp1 = ag.logpdf(data.f(ag.RowVecs(X1), data.s2), y1)
    l0 = eng.launch_count()
    lp2 = ag.logpdf(p1(ag.RowVecs(X2), s2v), y2)
    l_on = eng.launch_count() - l0
    eng.set_config(**AUTO_OFF)
    l0 = eng.launch_count()
    lp2_0 = ag.logpdf(p1(ag.RowVecs(X2), s2v), y2)
    l_off = eng.launch_count() - l0
    eng.set_config(**AUTO)
    assert l_on - l_off == _chol_delta(8320)[0], (l_on, l_off)  # n_pad = 1024: the substitution is on the tile path
    lp_all = ag.logpdf(data.f(ag.RowVecs(data.X[:n]), noise), data.y[:n])
    print("chain rule", (lp1 + lp2 - lp_all) / abs(lp_all), (lp1 + lp2_0 - lp_all) / abs(lp_all))
    # log p(y1, y2) = log p(y1) + log p(y2 | y1): the two sides differ by the rounding of two factorisations of 9200
    # points, each a few eps * cond(C) ~ 1e-16 * 1e5 relative in the logdet and the quadratic form
    assert abs(lp1 + lp2 - lp_all) <= 1e-9 * abs(lp_all), (lp1, lp2, lp_all)
    assert abs(lp1 + lp2_0 - lp_all) <= 1e-9 * abs(lp_all)


def test_extend_auto_fp32(ag, eng):
    """fp32, automatic policy: n1 = 900, n2 = 4200 (n2_pad = 4224 >= 4096: the int8-slice Cholesky with 512-wide panels;
    tensor mode 0 also narrows the panels to 128, so only the inequality of the counts is asserted)"""
    n1, n2 = 900, 4200
    data = Data(ag, np.float32, n1 + n2)
    p1, p2, p2_0, noise, l_on, l_off = _extend(ag, eng, data, n1, n2, AUTO, AUTO_OFF)
    assert l_on != l_off, l_on
    n, n_pad = n1 + n2, 1024 + 4224
    pr = data.oracle(n, noise)
    tol = _Tol32(pr, 0.05)
    print("A fp32 cond", tol.cond)
    _check_handle(p2, pr, n, tol, export=True, tag="A auto fp32")
    _check_handle(p2_0, pr, n, tol, export=False)
    _check_predictions(ag, eng, p2, pr, data, n_pad, AUTO, AUTO_OFF, tol, tag="A auto fp32")


# ---- B: logpdf and rand over the posterior (post_cond_impl) -----------------------------------------------------------
@pytest.mark.parametrize("dtype,m,mode", [(np.float64, 1300, "forced"), (np.float64, 2304, "forced"),
                                          (np.float64, 8320, "auto"), (np.float32, 4224, "auto")])
def test_post_cond(ag, eng, dtype, m, mode):
    """n = 2500 (n_pad = 2560 >= 2048: V = L^-1 K(x, x*) on the tensor substitution), then the M x M Cholesky of
    K** + S* - V'V on int8 panels"""
    on, off = (FORCED, FORCED_OFF) if mode == "forced" else (AUTO, AUTO_OFF)
    n = 2500
    data = Data(ag, dtype, n)
    eng.set_config(**on)
    post = ag.posterior(data.f(ag.RowVecs(data.X), data.s2), data.y)
    pr = data.oracle(n, np.full(n, data.s2))
    Xs = np.random.default_rng(m).random((m, data.X.shape[1])).astype(dtype)
    _check_post_cond(ag, eng, post, pr, data, Xs, 2560, on, off, _tol(dtype, pr, data.s2), tag="B %s %s" % (np.dtype(dtype).name, mode))


# ---- C: mean_and_cov and the solves on a plain fitted handle -----------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_plain_handle_mean_cov_and_solves(ag, eng, dtype):
    """n = 3000 (n_pad = 3072), mean_and_cov at M = 1024 and the operator API with 512 columns on the tensor substitution"""
    n = 3000
    data = Data(ag, dtype, n)
    post = ag.posterior(data.f(ag.RowVecs(data.X), data.s2), data.y)
    pr = data.oracle(n, np.full(n, data.s2))
    tol = _tol(dtype, pr, data.s2)
    _check_handle(post, pr, n, tol, export=False, tag="C %s" % np.dtype(dtype).name)
    _check_predictions(ag, eng, post, pr, data, 3072, AUTO, AUTO_OFF, tol, n_cov=1024, tag="C %s" % np.dtype(dtype).name)


# ---- D: not positive definite on the int8 path -------------------------------------------------------------------------
def _dpotrf_info(Cm):
    return int(lapack.dpotrf(Cm, lower=0, overwrite_a=1)[1])


def test_not_posdef_extension_on_int8_panels(ag, eng):
    """forced fp64, n1 = 700, n2 = 1300, noise -5 on new point 1100: its pivot is in the third outer panel, after two int8
    trailing updates.  PosDefException.info is the first failing pivot dpotrf reports on the batch matrix, in both modes;
    p1 still answers bit for bit and the engine still extends."""
    n1, n2, j = 700, 1300, 1100
    data = Data(ag, np.float64, n1 + n2)
    eng.set_config(**FORCED)
    p1 = ag.posterior(data.f(ag.RowVecs(data.X[:n1]), data.s2), data.y[:n1])
    m1, v1 = ag.mean_and_var(p1, ag.RowVecs(data.Xs[:300]))
    bad = data.nv[n1:].copy()
    bad[j] = -5.0
    Cm = ref.kernelmatrix(data.ks, data.X)
    Cm[np.diag_indices(n1 + n2)] += np.concatenate([np.full(n1, data.s2), bad])
    want = _dpotrf_info(Cm)
    assert n1 < want <= n1 + j + 1, want
    X2, y2 = data.seg(n1, n1 + n2)
    for cfg in (FORCED, FORCED_OFF):
        eng.set_config(**cfg)
        with pytest.raises(ag.PosDefException) as e:
            ag.posterior(p1(ag.RowVecs(X2), bad), y2)
        assert e.value.info == want, (cfg, e.value.info, want)
    eng.set_config(**FORCED)
    m1b, v1b = ag.mean_and_var(p1, ag.RowVecs(data.Xs[:300]))
    assert np.array_equal(m1, m1b) and np.array_equal(v1, v1b)
    p2 = ag.posterior(p1(ag.RowVecs(X2), data.nv[n1:]), y2)
    pr = data.oracle(n1 + n2, np.concatenate([np.full(n1, data.s2), data.nv[n1:].astype(np.float64)]))
    assert np.allclose(p2.data.alpha, pr["alpha"], **_Tol64.alpha(None, pr["alpha"]))


def test_not_posdef_post_cond_on_int8_panels(ag, eng):
    """the same for logpdf and rand over p1 at M = 2304 (the M x M Cholesky on four int8 panels): info is dpotrf's first
    failing pivot of C* + S*"""
    n1, m, j = 700, 2304, 1100
    data = Data(ag, np.float64, n1)
    eng.set_config(**FORCED)
    p1 = ag.posterior(data.f(ag.RowVecs(data.X), data.s2), data.y)
    pr = data.oracle(n1, np.full(n1, data.s2))
    Xs = np.random.default_rng(m).random((m, data.X.shape[1]))
    m1, v1 = ag.mean_and_var(p1, ag.RowVecs(Xs[:300]))
    bad = np.full(m, 0.05)
    bad[j] = -5.0
    _, Cs = ref.post_mean_and_cov(pr, Xs)
    Cs[np.diag_indices(m)] += bad
    want = _dpotrf_info(Cs)
    assert 0 < want <= j + 1, want
    fx = p1(ag.RowVecs(Xs), bad)
    for cfg in (FORCED, FORCED_OFF):
        eng.set_config(**cfg)
        for call in (lambda: ag.logpdf(fx, np.zeros(m)), lambda: ag.rand_from_normals(fx, np.zeros((m, 2)))):
            with pytest.raises(ag.PosDefException) as e:
                call()
            assert e.value.info == want, (cfg, e.value.info, want)
    eng.set_config(**FORCED)
    m1b, v1b = ag.mean_and_var(p1, ag.RowVecs(Xs[:300]))
    assert np.array_equal(m1, m1b) and np.array_equal(v1, v1b)
    ok = p1(ag.RowVecs(Xs), 0.05)
    Y = np.zeros(m)
    mo, Uo = _cond_oracle(pr, Xs, 0.05)
    want_lp = -0.5 * (m * ref.LOG2PI + ref.logdet_chol(Uo) + ref.tr_Xt_invA_X(Uo, Y - mo))
    assert _rel(ag.logpdf(ok, Y), want_lp) <= 1e-8


# ---- E: the slice workspace across handles of other sizes --------------------------------------------------------------
def test_slice_workspace_reuse_across_sizes(ag, eng):
    """one engine, forced int8 panels: post_cond at M = 2304 on an n = 2500 handle; mean_and_var at 1536 points on an
    n = 9200 extended handle (the workspace grows for its Schur Cholesky and its substitution); post_cond at M = 1300; the
    first call again.  The repeated call gives the same bits: nothing stale from a resize reaches it."""
    eng.set_config(**FORCED)
    data = Data(ag, np.float64, 2500)
    post = ag.posterior(data.f(ag.RowVecs(data.X), data.s2), data.y)
    rng = np.random.default_rng(17)
    Xa, Xb = rng.random((2304, 8)), rng.random((1300, 8))
    Za = np.asfortranarray(rng.standard_normal((2304, 4)))
    Zb = np.asfortranarray(rng.standard_normal((1300, 4)))
    first = ag.rand_from_normals(post(ag.RowVecs(Xa), 0.05), Za)
    big = Data(ag, np.float64, 9200)
    q1 = ag.posterior(big.f(ag.RowVecs(big.X[:1000]), big.s2), big.y[:1000])
    q2 = ag.posterior(q1(ag.RowVecs(big.X[1000:]), big.nv[1000:]), big.y[1000:])
    mu, v = ag.mean_and_var(q2, ag.RowVecs(big.Xs))
    assert np.all(np.isfinite(mu)) and np.all(np.isfinite(v))
    del q1, q2
    ag.rand_from_normals(post(ag.RowVecs(Xb), 0.05), Zb)
    again = ag.rand_from_normals(post(ag.RowVecs(Xa), 0.05), Za)
    assert np.array_equal(first, again)
