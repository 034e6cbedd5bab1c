"""The pullback of mean_and_var over an exact posterior on the device (agp_post_mean_var_grad), in fp64 and fp32: against
the CPU model tests/post_mean_var_grad_ref.py for the five single-kernel families under every transform in the row, column
and vector containers, per-point noises and vector means, composites (with Linear and Periodic factors) and the Mauna Loa
kernel on a train / held-out split of the CO2 data; the values against agp_post_mean_var; central differences of
agp_post_mean_var over x* and over refits; the test-side-only call (its x* gradient bit for bit, and no stacked pass,
from the launch counter); the backward substitution on its tile and int8-slice schedules, the branch asserted from the
launch counter; device memory, determinism, NULL outputs and cotangents, the error codes; and an L-BFGS-B replay of
analytic expected improvement maximised over x* with the test-side-only gradient.
Tolerances: rtol 1e-7 (fp64) / 2e-2 (fp32, against the model on the fp32-rounded inputs), atol the same times max|g|.  The
fp32 x* gradient is a sum over the training points of Kbar_sx[j, n] d1k(x*_j, x_n), whose weights carry the fp32 error of
alpha and P (relative, growing with cond(C)); its error is therefore bounded by that relative error times the sum of the
terms' magnitudes sum_n |Kbar_sx[j, n] d1k(x*_j, x_n)| + 2 |vbar_j d1k(x*_j, x*_j)|, and it is held to rtol times that
sum (xs_terms below), entry by entry."""
import ctypes as C

import numpy as np
import pytest
from scipy.stats import norm

import composite_ref as cr
import grad_x_ref as gx
import post_mean_var_grad_ref as pmv
from oracle import agp_ref as ref
from test_gpu_composite import KERNELS, _co2, _mauna_loa_kernel, oracle_of
from test_gpu_post_rand_grad import close_sum, f64
from test_gpu_rand_grad import _DevArr, _launches, check_single, close, container, kernel, x_rows

pytestmark = pytest.mark.gpu
RT = {np.float64: 1e-7, np.float32: 2e-2}
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]
TILE = 128


def data(N, M, D, dtype, seed=0):
    rng = np.random.default_rng(seed + 7 * N + 3 * M + D)
    return (rng.uniform(-2, 2, (N, D)).astype(dtype), rng.standard_normal(N).astype(dtype),
            rng.uniform(-2.2, 2.2, (M, D)).astype(dtype), rng.standard_normal(M).astype(dtype),
            rng.standard_normal(M).astype(dtype))


def xs_terms(k, X, Xs, mbar, vbar, alpha_P):
    """sum_n |Kbar_sx[j, n] d1k(x*_j, x_n)_d| + 2 |vbar_j d1k(x*_j, x*_j)_d| (M x D), the scale of the fp32 x* bound"""
    alpha, P = alpha_P
    Kbar = np.outer(mbar, alpha) - 2.0 * vbar[:, None] * P.T
    M = Xs.shape[0]
    d1 = gx.kernel_d1(k, Xs, Xs)[np.arange(M), np.arange(M)]
    return np.einsum("mi,mid->md", np.abs(Kbar), np.abs(gx.kernel_d1(k, Xs, X))) + 2.0 * np.abs(vbar)[:, None] * np.abs(d1)


def alpha_P(k, mean, noise, X, y, Xs):
    from scipy.linalg import cho_factor, cho_solve
    kc = gx.as_composite(k)
    N = X.shape[0]
    cf = cho_factor(cr.kernelmatrix(kc, X) + np.diag(noise.diag(N, np.float64)), lower=True)
    return cho_solve(cf, y - mean.vector(N, np.float64)), cho_solve(cf, cr.kernelmatrix(kc, X, Xs))


def close_xs(got, want, terms, rt):
    got = np.asarray(got, dtype=np.float64)
    assert np.all(np.isfinite(got))
    assert np.all(np.abs(got - want) <= rt * (np.abs(want) + terms) + 1e-300), np.max(np.abs(got - want) / (terms + 1e-300))


def fp32_eps(N, var, s2):
    """the relative error of alpha and P on an fp32 handle: 2^-24 cond(C), cond(C) <= 1 + N var / s2 (Gershgorin: the
    eigenvalues of K_xx + s2 I lie in [s2, N var + s2]), times 4 for the two substitutions and the products"""
    return 4.0 * 2.0 ** -24 * (1.0 + N * var / s2)


def check_kernel_terms(g, want, rt, eps):
    """fp32: each single-kernel entry is the sum of three block terms <Cbar, dK_xx> + <Kbar_sx, dK_sx> + <Sigmabar, dK_ss>
    that cancel (the means barely depend on the kernel variance: at N = 63, M = 17 the terms are ~50x the sum), so its
    rounding error is eps times the terms' magnitudes (the model's grad_abs), not a fraction of the sum"""
    for key, sl in [("variance", 0), ("scale", 1), ("ard", slice(5, None)), ("linear_c", 2)]:
        if key in g:
            got, w, a = (np.asarray(v, dtype=np.float64) for v in (g[key], want["grad"][sl], want["grad_abs"][sl]))
            assert np.all(np.abs(got - w) <= rt * np.abs(w) + eps * a), (key, got, w, a, eps)


def check_all(mv, g, want, spec, kind, rt, kernel=True, terms=None, eps=None):
    close(mv[0], want["mean"], rt)
    close(mv[1], want["var"], rt)
    if kernel and eps is None:
        check_single(g, want, spec, rt)
    elif kernel:
        check_kernel_terms(g, want, rt, eps)
    close_sum(g["noise"], want["grad"][3], want["noise_diag"], rt)
    close_sum(g["mean_c"], want["grad"][4], np.concatenate([want["mean_s_diag"], want["y"]]), rt)
    close(g["y"], want["y"], rt)
    close(x_rows(g["x"], kind), want["x"], rt)
    if terms is None:
        close(x_rows(g["xs"], kind), want["xs"], rt)
    else:
        close_xs(x_rows(g["xs"], kind), want["xs"], terms, rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_matches_model(ag, family, transform, dtype):
    rt = RT[dtype]
    for N, M, D, kind in [(1, 1, 1, "vec"), (63, 17, 3, "row"), (333, 129, 1, "col"), (333, 200, 40, "row"),
                          (1300, 1000, 3, "col")]:
        k, spec = kernel(ag, family, transform, D)
        X, y, Xs, mb, vb = data(N, M, D, dtype)
        p = ag.posterior(ag.GP(0.3, k)(container(ag, X, kind), 0.1), y)
        fx = p(container(ag, Xs, kind), 0.05)
        mv, g = ag.posterior_mean_var_grad(fx, mb, vb, inputs=True)
        args = (spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs), ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.05))
        want = pmv.post_mean_var_grad(*args, *f64(mb, vb))
        assert g["xs"].dtype == dtype and g["y"].dtype == dtype
        # the values are agp_post_mean_var's, bit for bit
        m2, v2 = ag.mean_and_var(fx)
        assert mv[0].tobytes() == m2.tobytes() and mv[1].tobytes() == v2.tobytes()
        terms = None
        if dtype == np.float32:
            X64, y64, Xs64 = f64(X, y, Xs)
            terms = xs_terms(spec, X64, Xs64, *f64(mb, vb), alpha_P(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X64, y64,
                                                                     Xs64))
        # fp32 Linear kernel gradients are differences of nearly equal terms (the posterior covariance of a rank-D prior is
        # the test noise plus O(D / N)), as for the held-out gradient (DESIGN s6): held to the model in fp64 only
        linear32 = spec.family == cr.LINEAR and dtype == np.float32
        check_all(mv, g, want, spec, kind, rt, kernel=not linear32, terms=terms,
                  eps=fp32_eps(N, 1.3, 0.1) if dtype == np.float32 else None)
        np.testing.assert_array_equal(g["noise_s"], np.sum(vb.astype(np.float64)))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_per_point_noises_and_vector_means(ag, dtype):
    N, M, D = 500, 300, 2
    k, spec = kernel(ag, cr.MATERN32, cr.T_ARD, D)
    X, y, Xs, mb, vb = data(N, M, D, dtype, seed=2)
    rng = np.random.default_rng(2)
    s2, s2s = rng.uniform(0.05, 0.2, N), rng.uniform(0.02, 0.1, M)
    p = ag.posterior(ag.GP(ag.CustomMean(lambda x: np.sin(x[0])), k)(ag.RowVecs(X), s2), y)
    mv, g = ag.posterior_mean_var_grad(p(ag.RowVecs(Xs), s2s), mb, vb, inputs=True)
    r = lambda a: np.asarray(a).astype(dtype).astype(np.float64)  # noqa: E731
    X64, Xs64 = f64(X, Xs)
    want = pmv.post_mean_var_grad(spec, ref.MeanSpec(2, v=r(np.sin(X64[:, 0]))), ref.NoiseSpec(1, v=r(s2)), X64, *f64(y),
                                  Xs64, ref.MeanSpec(2, v=r(np.sin(Xs64[:, 0]))), ref.NoiseSpec(1, v=r(s2s)), *f64(mb, vb))
    rt = RT[dtype]
    close(mv[0], want["mean"], rt)
    close(mv[1], want["var"], rt)
    for key, wk in [("noise", "noise_diag"), ("mean_v", "mean_diag"), ("noise_s", "noise_s_diag"),
                    ("mean_s_v", "mean_s_diag"), ("x", "x"), ("xs", "xs"), ("y", "y")]:
        close(g[key], want[wk], rt)
    if dtype == np.float32:
        check_kernel_terms(g, want, rt, fp32_eps(N, 1.3, 0.05))
    else:
        check_single(g, want, spec, rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname,D", [("stationary", 1), ("ard", 3), ("mixed", 3)])
def test_composite(ag, dtype, kname, D):
    k = KERNELS[kname](ag, D)
    ko = oracle_of(ag, k, D)
    X, y, Xs, mb, vb = data(333, 150, D, dtype, seed=6)
    p = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    mv, g = ag.posterior_mean_var_grad(p(ag.RowVecs(Xs), 0.05), mb, vb, inputs=True)
    want = pmv.post_mean_var_grad(ko, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs), ref.MeanSpec(1, 0.3),
                                  ref.NoiseSpec(0, 0.05), *f64(mb, vb))
    rt = RT[dtype]
    wk = ag.api._Flat(k, D).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(v, dtype=np.float64)).max() for v in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(np.asarray(a, dtype=np.float64), b, rtol=rt, atol=rt * scale)
    for key in ("x", "xs", "y"):
        close(g[key], want[key], rt)
    close(g["noise"], want["grad"][3], rt)
    close(g["mean_c"], want["grad"][4], rt)
    close(mv[0], want["mean"], rt)
    close(mv[1], want["var"], rt)


def test_linear_in_a_product_kdiag(ag):
    """a Linear factor inside a product and an ARD Linear alone: the kdiag term of the x* gradient, against the model with
    vbar only, and the mbar-only call for the cross pairs alone"""
    D, N, M = 2, 400, 70
    k = (0.7 * ag.LinearKernel(c=0.3) * ag.with_lengthscale(ag.SqExponentialKernel(), 1 / 0.6)
         + 0.4 * ag.LinearKernel(c=0.2).compose(ag.ARDTransform(np.array([0.8, 1.1]))) + ag.Matern32Kernel())
    ko = oracle_of(ag, k, D)
    X, y, Xs, mb, vb = data(N, M, D, np.float64, seed=13)
    p = ag.posterior(ag.GP(k)(ag.RowVecs(0.5 * X), 0.1), y)
    for m_, v_ in [(mb, vb), (None, vb), (mb, None)]:
        _, g = ag.posterior_mean_var_grad(p(ag.RowVecs(0.5 * Xs), 0.05), m_, v_, inputs=True, training=False)
        want = pmv.post_mean_var_grad(ko, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), 0.5 * X, y, 0.5 * Xs, ref.MeanSpec(),
                                      ref.NoiseSpec(0, 0.05), np.zeros(M) if m_ is None else m_,
                                      np.zeros(M) if v_ is None else v_)
        close(g["xs"], want["xs"], 1e-7)


def test_mauna_loa_forecast(ag):
    """the Mauna Loa kernel on the CO2 data: train on the first 400 months, predict the next 150"""
    x, y = _co2()
    xtr, ytr, xte = x[:400], y[:400], x[400:550]
    k = _mauna_loa_kernel(ag, np.array([4.0, 4.0, 0.0, 1.0, 4.0, 0.0, 0.0, -1.0, -2.0, -2.0, -2.0]))
    ko = oracle_of(ag, k, 1)
    m = float(np.mean(ytr))
    rng = np.random.default_rng(21)
    mb, vb = rng.standard_normal(150), rng.standard_normal(150)
    p = ag.posterior(ag.GP(m, k)(xtr, 0.05), ytr)
    mv, g = ag.posterior_mean_var_grad(p(xte, 0.05), mb, vb, inputs=True)
    want = pmv.post_mean_var_grad(ko, ref.MeanSpec(1, m), ref.NoiseSpec(0, 0.05), xtr[:, None], ytr, xte[:, None],
                                  ref.MeanSpec(1, m), ref.NoiseSpec(0, 0.05), mb, vb)
    wk = ag.api._Flat(k, 1).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(v, dtype=np.float64)).max() for v in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(a, b, rtol=1e-7, atol=1e-7 * scale)
    close(mv[0], want["mean"], 1e-9)
    close(mv[1], want["var"], 1e-7)
    close(g["x"], want["x"][:, 0], 1e-7)
    close(g["xs"], want["xs"][:, 0], 1e-7)
    close(g["noise"], want["grad"][3], 1e-7)
    close(g["mean_c"], want["grad"][4], 1e-7)
    close(g["y"], want["y"], 1e-7)


def test_central_differences(ag):
    """x* against central differences of agp_post_mean_var; the kernel scale, the training noise, an input and a target
    against central differences over refits"""
    N, M, D = 120, 40, 2
    X, y, Xs, mb, vb = data(N, M, D, np.float64, seed=11)
    ls, s2 = 0.9, 0.1

    def F(ls_=ls, s2_=s2, X_=X, y_=y, Xs_=Xs):
        k = ag.with_lengthscale(ag.Matern52Kernel(), ls_)
        p = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X_), s2_), y_)
        m, v = ag.mean_and_var(p(ag.RowVecs(Xs_), 0.05))
        return float(np.dot(mb, m) + np.dot(vb, v))
    p = ag.posterior(ag.GP(0.3, ag.with_lengthscale(ag.Matern52Kernel(), ls))(ag.RowVecs(X), s2), y)
    _, g = ag.posterior_mean_var_grad(p(ag.RowVecs(Xs), 0.05), mb, vb, inputs=True)
    _, gt = ag.posterior_mean_var_grad(p(ag.RowVecs(Xs), 0.05), mb, vb, inputs=True, training=False)
    h = 1e-5
    fd = lambda a, b: (a - b) / (2 * h)  # noqa: E731
    s = 1.0 / ls
    d_ls = fd(F(ls_=1.0 / (s + h)), F(ls_=1.0 / (s - h)))
    assert abs(g["scale"] - d_ls) <= 1e-6 * max(1.0, abs(d_ls)), (g["scale"], d_ls)
    d_s2 = fd(F(s2_=s2 + h), F(s2_=s2 - h))
    assert abs(g["noise"] - d_s2) <= 1e-6 * max(1.0, abs(d_s2)), (g["noise"], d_s2)
    for i, d in [(3, 0), (77, 1)]:
        Xp, Xm = X.copy(), X.copy()
        Xp[i, d] += h
        Xm[i, d] -= h
        v = fd(F(X_=Xp), F(X_=Xm))
        assert abs(g["x"][i, d] - v) <= 1e-6 * max(1.0, abs(v)), (i, d, g["x"][i, d], v)
    for j, d in [(0, 0), (17, 1), (39, 0)]:
        Xsp, Xsm = Xs.copy(), Xs.copy()
        Xsp[j, d] += h
        Xsm[j, d] -= h
        v = fd(F(Xs_=Xsp), F(Xs_=Xsm))
        assert abs(g["xs"][j, d] - v) <= 1e-6 * max(1.0, abs(v)), (j, d, g["xs"][j, d], v)
        assert gt["xs"][j, d] == g["xs"][j, d]
    yp, ym = y.copy(), y.copy()
    yp[10] += h
    ym[10] -= h
    v = fd(F(y_=yp), F(y_=ym))
    assert abs(g["y"][10] - v) <= 1e-6 * max(1.0, abs(v)), (g["y"][10], v)


@pytest.mark.parametrize("family", [cr.SE, cr.MATERN12])
def test_test_point_on_a_training_point(ag, family):
    """x*_0 = x_5: the pair adds exactly 0 (Matern 1/2: the zero subgradient); the result is finite and the model's"""
    N, M, D = 90, 6, 2
    k, spec = kernel(ag, family, cr.T_SCALE, D)
    X, y, Xs, mb, vb = data(N, M, D, np.float64, seed=14)
    Xs[0] = X[5]
    p = ag.posterior(ag.GP(k)(ag.RowVecs(X), 0.1), y)
    _, g = ag.posterior_mean_var_grad(p(ag.RowVecs(Xs), 0.05), mb, vb, inputs=True, training=False)
    want = pmv.post_mean_var_grad(spec, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, y, Xs, ref.MeanSpec(), ref.NoiseSpec(0, 0.05),
                                  mb, vb)
    close(g["xs"], want["xs"], 1e-7)


# ---- the raw entry point on a handle -----------------------------------------------------------------------------------
def _call(ag, h, Xs, mb, vb, outs=None, layout=0, M=None):
    eng = ag.engine()
    p = lambda a: a if isinstance(a, int) else ag._cabi.ptr(a)  # noqa: E731
    dp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    o = outs or {}
    M = (Xs.shape[0] if layout == 0 else Xs.shape[-1]) if M is None else M
    return eng.L.agp_post_mean_var_grad(h, layout, p(Xs), M, p(mb), p(vb), dp(o.get("g")), p(o.get("nd")), p(o.get("md")),
                                        p(o.get("yb")), p(o.get("xg")), p(o.get("xsg")))


def _outs(N, M, D, dtype, glen=None):
    e = lambda *s: np.empty(s, dtype=dtype)  # noqa: E731
    # the input gradients point-major: n x D row-major
    return dict(g=np.zeros(5 + D if glen is None else glen), nd=e(N), md=e(N), yb=e(N), xg=e(N, D), xsg=e(M, D))


def _mean_var_launches(ag, h, Xs, M, dtype):
    """launches of agp_post_mean_var with the variances on the same handle and points"""
    eng = ag.engine()
    m, v = np.empty(M, dtype=dtype), np.empty(M, dtype=dtype)
    n, rc = _launches(ag, lambda: eng.L.agp_post_mean_var(h, 0, ag._cabi.ptr(Xs), M, None, None, ag._cabi.ptr(m),
                                                          ag._cabi.ptr(v)))
    assert rc == 0
    return n


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_test_side_only_call(ag, dtype):
    """xs_grad_out alone: the same bits as in the full call, and the launches of agp_post_mean_var's forward plus the
    backward substitution and the two cross kernels -- one more than y_bar alone (its GEMV), none of the stacked pass"""
    N, M, D = 700, 300, 3
    k, _ = kernel(ag, cr.MATERN32, cr.T_SCALE, D)
    X, y, Xs, mb, vb = data(N, M, D, dtype, seed=7)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Xsc = post.data.C.h, np.ascontiguousarray(Xs)
    o = _outs(N, M, D, dtype)
    n_full, rc = _launches(ag, lambda: _call(ag, h, Xsc, mb, vb, outs=o))
    assert rc == 0
    xs = dict(xsg=np.empty((M, D), dtype=dtype))
    n_xs, rc = _launches(ag, lambda: _call(ag, h, Xsc, mb, vb, outs=xs))
    assert rc == 0
    assert xs["xsg"].tobytes() == o["xsg"].tobytes()
    yo = dict(yb=np.empty(N, dtype=dtype))
    n_y, rc = _launches(ag, lambda: _call(ag, h, Xsc, mb, vb, outs=yo))
    assert rc == 0 and yo["yb"].tobytes() == o["yb"].tobytes()
    assert n_xs == n_y + 1, (n_xs, n_y)
    assert n_full - n_xs >= 4, (n_full, n_xs)  # the stacked pass: Kbar_sx and Cbar GEMMs, the reductions
    nblk = -(-N // TILE)
    d = n_xs - _mean_var_launches(ag, h, Xsc, M, dtype)  # the backward substitution + 2 - (kdiag, gemv, colsumsq)
    assert abs(d - (2 * nblk - 2)) <= 2, (d, nblk)


def _subst_case(ag, dtype, N, M, key, mode, int8):
    """the fit and the calls under `key` = mode, then again under 0 (the tile kernels).  The launches of the backward
    substitution are those of the test-side-only call minus agp_post_mean_var's on the same points (the same forward
    substitution): on the tile schedule 2 nblk - 1 GEMMs (2 nblk - 2 after the difference), and the int8-slice schedule
    differs from it.  M = 1 stays on the tile schedule (fewer than 512 columns) and one row block of the cross pass is
    split over the training points.  Both agree with the model."""
    eng = ag.engine()
    D = 2
    k, spec = kernel(ag, cr.SE, cr.T_ARD, D)
    X, y, Xs, mb, vb = data(N, M, D, dtype, seed=12)
    Xsc = np.ascontiguousarray(Xs)
    nblk = -(-N // TILE)
    cfg = eng.get_config()
    res = []
    try:
        for m in (mode, 0):
            eng.set_config(**{key: m})  # before the fit: the handle's own factor comes from this policy too
            post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
            h = post.data.C.h
            n_xs, rc = _launches(ag, lambda: _call(ag, h, Xsc, mb, vb, outs=dict(xsg=np.empty((M, D), dtype=dtype))))
            assert rc == 0
            d = n_xs - _mean_var_launches(ag, h, Xsc, M, dtype)
            o = _outs(N, M, D, dtype)
            assert _call(ag, h, Xsc, mb, vb, outs=o) == 0
            res.append((d, o))
    finally:
        eng.set_config(**{key: getattr(cfg, key)})
    tc, tile = res[0][0], res[1][0]
    assert abs(tile - (2 * nblk - 2)) <= 2, (tile, nblk)
    assert (tc != tile) == int8, (tc, tile)
    want = pmv.post_mean_var_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs), ref.MeanSpec(1, 0.3),
                                  ref.NoiseSpec(0, 0.05), *f64(mb, vb))
    rt = RT[dtype]
    for _, o in res:
        for key_, wk in [("nd", "noise_diag"), ("yb", "y"), ("md", "mean_diag"), ("xg", "x"), ("xsg", "xs")]:
            close(o[key_], want[wk], rt)
        close(o["g"][[0, 5, 6]], want["grad"][[0, 5, 6]], rt)
        close_sum(o["g"][3], want["grad"][3], want["noise_diag"], rt)
        close_sum(o["g"][4], want["grad"][4], np.concatenate([want["mean_s_diag"], want["y"]]), rt)


def test_backward_substitution_forced_fp64(ag):
    """fp64 at N = 2304, M = 512 with the int8-slice kernels forced (fp64_mode = 1)"""
    _subst_case(ag, np.float64, 2304, 512, "fp64_mode", 1, True)


@pytest.mark.parametrize("M,int8", [(600, True), (1, False)])
@pytest.mark.parametrize("dtype,N,key", [(np.float64, 8320, "fp64_mode"), (np.float32, 4224, "fp32_mode")])
def test_backward_substitution_automatic(ag, dtype, N, key, M, int8):
    """fp64 N = 8320 and fp32 N = 4224: the automatic policy (-1) takes the int8-slice kernels at M = 600, the tile
    kernels at M = 1"""
    _subst_case(ag, dtype, N, M, key, -1, int8)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_determinism_null_outputs_and_layouts(ag, dtype):
    N, M, D = 700, 300, 3
    k, _ = kernel(ag, cr.MATERN32, cr.T_SCALE, D)
    X, y, Xs, mb, vb = data(N, M, D, dtype, seed=7)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Xsc = post.data.C.h, np.ascontiguousarray(Xs)
    outs = []
    for _ in range(2):
        o = _outs(N, M, D, dtype)
        assert _call(ag, h, Xsc, mb, vb, outs=o) == 0
        outs.append(o)
    for key in outs[0]:
        if key != "g":
            assert outs[0][key].tobytes() == outs[1][key].tobytes(), key
    assert outs[0]["g"][3:5].tobytes() == outs[1]["g"][3:5].tobytes()
    np.testing.assert_allclose(outs[0]["g"], outs[1]["g"], rtol=1e-10, atol=1e-10 * np.abs(outs[0]["g"]).max())
    for key in ("md", "yb", "nd", "xg", "xsg"):  # each alone: the rest of the work is skipped, the bits are the same
        o = {key: np.empty_like(outs[0][key])}
        assert _call(ag, h, Xsc, mb, vb, outs=o) == 0
        assert o[key].tobytes() == outs[0][key].tobytes(), key
    # feature-major: the input points and both input gradients as M x D / N x D column-major
    o = dict(xg=np.empty((N, D), dtype=dtype, order="F"), xsg=np.empty((M, D), dtype=dtype, order="F"))
    assert _call(ag, h, np.asfortranarray(Xs), mb, vb, outs=o, layout=1, M=M) == 0
    assert o["xg"].tobytes(order="F") == np.asfortranarray(outs[0]["xg"]).tobytes(order="F")
    assert o["xsg"].tobytes(order="F") == np.asfortranarray(outs[0]["xsg"]).tobytes(order="F")
    assert _call(ag, h, Xsc, mb, vb) == 0  # nothing requested
    # NULL cotangents are zeros
    z = np.zeros(M, dtype=dtype)
    for m_, v_ in [(None, vb), (mb, None), (None, None)]:
        a, b = _outs(N, M, D, dtype), _outs(N, M, D, dtype)
        assert _call(ag, h, Xsc, m_, v_, outs=a) == 0
        assert _call(ag, h, Xsc, z if m_ is None else m_, z if v_ is None else v_, outs=b) == 0
        for key in ("nd", "md", "yb", "xg", "xsg"):
            assert a[key].tobytes() == b[key].tobytes(), key
        np.testing.assert_allclose(a["g"], b["g"], rtol=1e-10, atol=1e-10 * max(np.abs(b["g"]).max(), 1e-300))
    assert np.all(a["xsg"] == 0) and np.all(a["yb"] == 0)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_device_memory(ag, dtype):
    torch = pytest.importorskip("torch")
    cabi = ag._cabi
    eng = ag.engine()
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    N, M, D = 500, 200, 4
    k, _ = kernel(ag, cr.SE, cr.T_ARD, D)
    X, y, Xs, mb, vb = data(N, M, D, dtype, seed=8)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Xsc = post.data.C.h, np.ascontiguousarray(Xs)
    o0 = _outs(N, M, D, dtype)
    assert _call(ag, h, Xsc, mb, vb, outs=o0) == 0
    Xd = torch.from_numpy(Xsc.ravel().copy()).cuda()
    mbd, vbd = torch.from_numpy(mb.copy()).cuda(), torch.from_numpy(vb.copy()).cuda()
    dev = {key: torch.empty(v.size, dtype=tdt, device="cuda") for key, v in o0.items() if key != "g"}
    o = {key: t.data_ptr() for key, t in dev.items()}
    o["g"] = np.zeros(5 + D)
    torch.cuda.synchronize()
    eng.set_memspace(cabi.AGP_MEM_DEVICE)
    try:
        rc = _call(ag, h, _DevArr(Xd, M, D), mbd.data_ptr(), vbd.data_ptr(), outs=o, M=M)
    finally:
        eng.set_memspace(cabi.AGP_MEM_HOST)
    assert rc == 0
    for key, t in dev.items():
        assert t.cpu().numpy().tobytes() == o0[key].tobytes(order="A"), key
    np.testing.assert_allclose(o["g"], o0["g"], rtol=1e-10, atol=1e-10 * np.abs(o0["g"]).max())


def test_errors(ag):
    cabi = ag._cabi
    N, M, D = 50, 20, 2
    k, _ = kernel(ag, cr.SE, cr.T_SCALE, D)
    X, y, Xs, mb, vb = data(N, M, D, np.float64, seed=9)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Xsc = post.data.C.h, np.ascontiguousarray(Xs)
    g = dict(g=np.zeros(5 + D))
    assert _call(ag, h, None, mb, vb, outs=g, M=M) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, mb, vb, outs=g, layout=2) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, mb, vb, outs=g, M=0) == cabi.AGP_ERR_DIM_MISMATCH
    assert _call(ag, h, Xsc, mb, vb, outs=g, M=-3) == cabi.AGP_ERR_DIM_MISMATCH
    assert ag.engine().L.agp_post_mean_var_grad(None, 0, cabi.ptr(Xsc), M, cabi.ptr(mb), cabi.ptr(vb),
                                                *([None] * 6)) == cabi.AGP_ERR_INVALID
    X2, y2, _, _, _ = data(20, 1, D, np.float64, seed=10)
    post2 = ag.posterior(post(ag.RowVecs(X2), 0.1), y2)
    assert _call(ag, post2.data.C.h, Xsc, mb, vb, outs=dict(xsg=np.empty((M, D)))) == cabi.AGP_ERR_UNSUPPORTED
    with pytest.raises(ag.AGPError):
        ag.posterior_mean_var_grad(post2(ag.RowVecs(Xs), 0.05), mb, vb)
    o = _outs(N, M, D, np.float64)  # the handle still works after every refusal
    assert _call(ag, h, Xsc, mb, vb, outs=o) == 0
    assert np.all(np.isfinite(o["g"])) and np.all(np.isfinite(o["xsg"]))


def test_lbfgs_expected_improvement_replay(ag):
    """analytic expected improvement EI(x*) = (mu - best) Phi(z) + sigma phi(z), z = (mu - best) / sigma, summed over
    q = 3 candidates and maximised by L-BFGS-B over x* with the test-side-only device gradient (training=False) and with
    the model's: the two paths agree and reach the same optimum.  Eight training points keep the posterior variance, and
    so the expected improvement away from them, large enough to move every candidate"""
    from scipy.optimize import minimize
    N, q = 8, 3
    rng = np.random.default_rng(17)
    X = rng.uniform(-2, 2, (N, 1))
    y = np.sin(2 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    best = float(np.max(y))
    k = 1.2 * ag.with_lengthscale(ag.SqExponentialKernel(), 0.6)
    spec = ref.KernelSpec(cr.SE, 1.2, cr.T_SCALE, 1.0 / 0.6)
    p = ag.posterior(ag.GP(k)(X[:, 0], 0.01), y)

    def ei_and_bars(mu, var):
        sd = np.sqrt(var)
        z = (mu - best) / sd
        return float(np.sum((mu - best) * norm.cdf(z) + sd * norm.pdf(z))), norm.cdf(z), norm.pdf(z) / (2.0 * sd)

    def dev(xs):
        fx = p(xs, 1e-9)
        v, mb, vb = ei_and_bars(*ag.mean_and_var(fx))
        _, g = ag.posterior_mean_var_grad(fx, mb, vb, inputs=True, training=False)
        return -v, -np.asarray(g["xs"], dtype=np.float64)

    def model(xs):
        args = (spec, ref.MeanSpec(), ref.NoiseSpec(0, 0.01), X, y, xs[:, None], ref.MeanSpec(), ref.NoiseSpec(0, 1e-9))
        r = pmv.post_mean_var_grad(*args, np.zeros(q), np.zeros(q))
        v, mb, vb = ei_and_bars(r["mean"], r["var"])
        return -v, -pmv.post_mean_var_grad(*args, mb, vb)["xs"][:, 0]
    x0 = np.array([-1.5, 0.2, 1.4])
    paths = []
    for fun in (dev, model):
        path = []
        res = minimize(fun, x0, jac=True, method="L-BFGS-B", bounds=[(-2, 2)] * q, callback=lambda t: path.append(t.copy()),
                       options=dict(maxiter=30))
        paths.append((np.array(path), res.x, res.fun))
    assert len(paths[0][0]) > 2
    n = min(len(paths[0][0]), len(paths[1][0]), 8)
    np.testing.assert_allclose(paths[0][0][:n], paths[1][0][:n], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(paths[0][1], paths[1][1], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(paths[0][2], paths[1][2], rtol=1e-8)
