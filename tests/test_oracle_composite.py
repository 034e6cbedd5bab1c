"""The CPU model of composite kernels (tests/composite_ref.py) pinned against implementations that share no code with it:
scikit-learn's kernels and GaussianProcessRegressor, 60-digit mpmath arithmetic, and central finite differences of its own
logpdf for the gradient.  scikit-learn and mpmath are required: a missing one fails these tests rather than skipping them."""
import numpy as np
import pytest

from oracle import agp_ref as ref
import composite_ref as cr


def _sk_pair(ell_se=1.3, ell_per=0.7, p=1.1, ell_se2=2.0, ell_rq=0.9, a_rq=1.7, c=0.6, sigma0=0.8):
    from sklearn.gaussian_process.kernels import RBF, ConstantKernel, DotProduct, ExpSineSquared, RationalQuadratic
    sk = (RBF(ell_se) + ExpSineSquared(ell_per, p) * RBF(ell_se2) + RationalQuadratic(ell_rq, a_rq)
          + ConstantKernel(c) * DotProduct(sigma0))
    k = cr.Composite([1.0, 1.0, 1.0, c], [
        [cr.Factor(cr.SE, cr.T_SCALE, 1 / ell_se)],
        [cr.Factor(cr.PERIODIC, cr.T_SCALE, 1 / p, r=np.array([ell_per / 2])), cr.Factor(cr.SE, cr.T_SCALE, 1 / ell_se2)],
        [cr.Factor(cr.RQ, cr.T_SCALE, 1 / ell_rq, param=a_rq)],
        [cr.Factor(cr.LINEAR, param=sigma0 ** 2)]])
    return sk, k


def test_kernelmatrix_matches_sklearn():
    rng = np.random.default_rng(0)
    X, Z = rng.normal(size=(40, 1)) * 2, rng.normal(size=(25, 1)) * 2
    sk, k = _sk_pair()
    np.testing.assert_allclose(cr.kernelmatrix(k, X), sk(X), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(cr.kernelmatrix(k, X, Z), sk(X, Z), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(cr.kernelmatrix_diag(k, X), sk.diag(X), rtol=1e-12, atol=1e-12)


def test_white_term_on_distinct_points_matches_sklearn():
    from sklearn.gaussian_process.kernels import RBF, WhiteKernel
    X = np.linspace(0, 3, 30)[:, None]  # distinct: sklearn's White is i == j, KernelFunctions' is x == x'
    sk = RBF(0.5) + WhiteKernel(0.3)
    k = cr.Composite([1.0, 0.3], [[cr.Factor(cr.SE, cr.T_SCALE, 2.0)], [cr.Factor(cr.WHITE)]])
    np.testing.assert_allclose(cr.kernelmatrix(k, X), sk(X), rtol=1e-12, atol=1e-12)


def test_lml_and_prediction_match_sklearn():
    from sklearn.gaussian_process import GaussianProcessRegressor
    rng = np.random.default_rng(1)
    X = np.sort(rng.uniform(0, 5, 60))[:, None]
    y = np.sin(3 * X[:, 0]) + 0.3 * X[:, 0] + 0.1 * rng.normal(size=60)
    Xs = np.linspace(-1, 6, 17)[:, None]
    sk, k = _sk_pair()
    s2 = 0.05
    gpr = GaussianProcessRegressor(sk, alpha=s2, optimizer=None, normalize_y=False).fit(X, y)
    noise = ref.NoiseSpec(0, s2)
    lp = cr.logpdf(k, ref.MeanSpec(), noise, X, y)
    assert abs(lp - gpr.log_marginal_likelihood_value_) <= 1e-10 * abs(lp)
    post = cr.posterior(k, ref.MeanSpec(), noise, X, y)
    m, v = cr.post_mean_and_var(post, Xs)
    ms, ss = gpr.predict(Xs, return_std=True)
    np.testing.assert_allclose(m, ms, rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(np.sqrt(np.maximum(v, 0)), ss, rtol=1e-7, atol=1e-9)


def test_logpdf_matches_mpmath_with_ard_periodic():
    import mpmath as mp
    mp.mp.dps = 60
    rng = np.random.default_rng(2)
    n, D = 12, 2
    X = rng.normal(size=(n, D))
    y = rng.normal(size=n)
    v, rr = np.array([0.7, 1.9]), np.array([0.8, 1.3])
    k = cr.Composite([1.3, 0.4], [[cr.Factor(cr.PERIODIC, cr.T_ARD, ard=v, r=rr), cr.Factor(cr.MATERN52, cr.T_SCALE, 0.6)],
                                  [cr.Factor(cr.RQ, cr.T_NONE, param=0.9)]])
    s2 = 0.1
    lp = cr.logpdf(k, ref.MeanSpec(), ref.NoiseSpec(0, s2), X, y)
    K = mp.matrix(n, n)
    for i in range(n):
        for j in range(n):
            xi, xj = [mp.mpf(float(a)) for a in X[i]], [mp.mpf(float(a)) for a in X[j]]
            per = mp.exp(-sum((mp.sin(mp.pi * mp.mpf(float(v[d])) * (xi[d] - xj[d])) / mp.mpf(float(rr[d]))) ** 2
                              for d in range(D)) / 2)
            r = mp.sqrt(sum((mp.mpf("0.6") * (xi[d] - xj[d])) ** 2 for d in range(D))) * mp.sqrt(5)
            m52 = (1 + r + r ** 2 / 3) * mp.exp(-r)
            d2 = sum((xi[d] - xj[d]) ** 2 for d in range(D))
            rq = (1 + d2 / (2 * mp.mpf("0.9"))) ** (-mp.mpf("0.9"))
            K[i, j] = mp.mpf("1.3") * per * m52 + mp.mpf("0.4") * rq + (mp.mpf(s2) if i == j else 0)
    yv = mp.matrix([mp.mpf(float(a)) for a in y])
    L = mp.cholesky(K)
    z = mp.lu_solve(L, yv)
    quad = sum(z[i] ** 2 for i in range(n))
    logdet = 2 * sum(mp.log(L[i, i]) for i in range(n))
    exact = -(n * mp.log(2 * mp.pi) + logdet + quad) / 2
    assert abs(lp - float(exact)) <= 1e-11 * abs(float(exact))


def _perturbable(k):
    """(get, set) pairs for every descriptor parameter, in the agp_post_logpdf_grad order"""
    out = []
    for t, fs in enumerate(k.factors):
        out.append((lambda k, t=t: k.variance[t], lambda k, x, t=t: k.variance.__setitem__(t, x)))
        for F in fs:
            if F.transform == cr.T_SCALE:
                out.append((lambda k, F=F: F.scale, lambda k, x, F=F: setattr(F, "scale", x)))
            elif F.transform == cr.T_ARD:
                for d in range(len(F.ard)):
                    out.append((lambda k, F=F, d=d: F.ard[d], lambda k, x, F=F, d=d: F.ard.__setitem__(d, x)))
            if F.family in (cr.RQ, cr.LINEAR, cr.CONSTANT):
                out.append((lambda k, F=F: F.param, lambda k, x, F=F: setattr(F, "param", x)))
            if F.family == cr.PERIODIC:
                for d in range(len(F.r)):
                    out.append((lambda k, F=F, d=d: F.r[d], lambda k, x, F=F, d=d: F.r.__setitem__(d, x)))
    return out


def fd_composite():
    D = 2
    return cr.Composite([1.2, 0.5, 0.3], [
        [cr.Factor(cr.PERIODIC, cr.T_SCALE, 0.8, r=np.array([0.9, 1.4])), cr.Factor(cr.SE, cr.T_ARD, ard=np.array([0.6, 1.1]))],
        [cr.Factor(cr.RQ, cr.T_SCALE, 1.3, param=1.5), cr.Factor(cr.CONSTANT, param=0.7)],
        [cr.Factor(cr.LINEAR, cr.T_ARD, ard=np.array([0.5, 0.9]), param=0.4), cr.Factor(cr.MATERN32, cr.T_SCALE, 0.7),
         cr.Factor(cr.PERIODIC, cr.T_ARD, ard=np.array([1.1, 0.6]), r=np.array([1.2, 0.8])),
         cr.Factor(cr.MATERN12, cr.T_NONE)]]), D


def test_oracle_gradient_matches_finite_differences():
    k, D = fd_composite()
    rng = np.random.default_rng(3)
    X = rng.normal(size=(30, D))
    y = rng.normal(size=30)
    noise, mean = ref.NoiseSpec(0, 0.2), ref.MeanSpec(1, 0.3)
    g, gn = cr.logpdf_grad(k, mean, noise, X, y)
    h = 1e-6
    for i, (get, set_) in enumerate(_perturbable(k)):
        x0 = get(k)
        set_(k, x0 + h)
        lp = cr.logpdf(k, mean, noise, X, y)
        set_(k, x0 - h)
        lm = cr.logpdf(k, mean, noise, X, y)
        set_(k, x0)
        fd = (lp - lm) / (2 * h)
        assert abs(g[5 + i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, g[5 + i], fd)
    fdn = (cr.logpdf(k, mean, ref.NoiseSpec(0, 0.2 + h), X, y) - cr.logpdf(k, mean, ref.NoiseSpec(0, 0.2 - h), X, y)) / (2 * h)
    assert abs(g[3] - fdn) <= 1e-6 * max(1.0, abs(fdn))
    fdm = (cr.logpdf(k, ref.MeanSpec(1, 0.3 + h), noise, X, y) - cr.logpdf(k, ref.MeanSpec(1, 0.3 - h), noise, X, y)) / (2 * h)
    assert abs(g[4] - fdm) <= 1e-6 * max(1.0, abs(fdm))
    assert np.all(g[:3] == 0)
