"""Composite kernels (sums of product terms) on the device, in fp64 and fp32, against the CPU model tests/composite_ref.py:
the Gram, the fit, the posterior's predictions, sampling and logpdf, sequential conditioning and the logpdf gradient; the
Mauna Loa example replayed through L-BFGS-B on the device's value and gradient; and the entry points that must decline a
composite kernel.  Tolerances: logpdf rtol 1e-8 (fp64) / 1e-4 (fp32), element-wise as tests/test_gpu_parity.py."""
import ctypes as C
import os

import numpy as np
import pytest

import composite_ref as cr
from oracle import agp_ref as ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def k_stationary(ag, D):
    """every distance family as a factor, with Scale transforms, White included (the Mauna Loa shape)"""
    SE = lambda s, l: s ** 2 * ag.with_lengthscale(ag.SqExponentialKernel(), l)  # noqa: E731
    per = ag.with_lengthscale(ag.PeriodicKernel(r=[0.6]), 1.3)
    rq = 0.7 ** 2 * ag.with_lengthscale(ag.RationalQuadraticKernel(alpha=0.8), 0.9 * np.sqrt(D))
    return (SE(1.2, 1.5 * np.sqrt(D)) + per * SE(0.8, 2.0 * np.sqrt(D)) + rq
            + (SE(0.3, 0.2 * np.sqrt(D)) + 0.2 ** 2 * ag.WhiteKernel()))


def k_ard(ag, D):
    """ARD on every family that has a distance, Linear and Constant, Matern 1/2 (Scale) and 5/2 (none): 6 accumulators"""
    rng = np.random.default_rng(D)
    v = lambda: rng.uniform(0.4, 1.2, D) / np.sqrt(D)  # noqa: E731
    return (ag.SqExponentialKernel().compose(ag.ARDTransform(v())) * ag.PeriodicKernel(r=rng.uniform(0.8, 1.5, D)).compose(
        ag.ARDTransform(v() * 0.5))
        + 0.5 * ag.RationalQuadraticKernel(alpha=1.3).compose(ag.ARDTransform(v()))
        + ag.LinearKernel(c=0.3).compose(ag.ARDTransform(v() * 0.3)) * ag.ConstantKernel(c=0.2)
        + 0.6 * ag.Matern32Kernel().compose(ag.ARDTransform(v()))
        + ag.with_lengthscale(ag.Matern12Kernel(), 2.0 * np.sqrt(D)) * ag.Matern52Kernel().compose(ag.ScaleTransform(0.5 / np.sqrt(D))))


def k_mixed(ag, D):
    """the combinations the other two leave out: Linear with Scale (the shared raw dot product and its scale gradient),
    White with Scale and with ARD, Matern 1/2 and 5/2 with ARD: 4 terms, 5 factors, 5 accumulators"""
    rng = np.random.default_rng(100 + D)
    v = lambda: rng.uniform(0.4, 1.2, D) / np.sqrt(D)  # noqa: E731
    return (0.5 * ag.with_lengthscale(ag.LinearKernel(c=0.2), 2.0 * np.sqrt(D)) * ag.Matern12Kernel().compose(ag.ARDTransform(v()))
            + 0.8 * ag.Matern52Kernel().compose(ag.ARDTransform(v()))
            + 0.1 * ag.WhiteKernel().compose(ag.ScaleTransform(0.5))
            + 0.05 * ag.WhiteKernel().compose(ag.ARDTransform(v())))


KERNELS = {"stationary": k_stationary, "ard": k_ard, "mixed": k_mixed}


def oracle_of(ag, k, D):
    keep = []
    ks = ag.api._Flat(k, D).struct(np.float64, keep)
    return cr.from_struct(ks, D, np.float64)


def data(N, D, dtype, seed=0, dup=True):
    rng = np.random.default_rng(seed + 7 * N + D)
    X = rng.uniform(-2, 2, (N, D))
    if dup and N > 4:  # exact duplicates: the White factor must see x == x' off the diagonal
        X[N // 2] = X[1]
        X[N - 1] = X[0]
    y = np.sin(2 * X).sum(1) + 0.1 * rng.normal(size=N)
    X = X.astype(dtype)
    return X, y.astype(dtype), X.astype(np.float64)


TOL = {np.float64: dict(rtol=1e-8, el=1e-7), np.float32: dict(rtol=1e-4, el=5e-3)}


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname", ["stationary", "ard", "mixed"])
@pytest.mark.parametrize("N,D", [(1, 1), (63, 3), (333, 1), (333, 40), (1300, 1), (1300, 3)])
def test_composite_parity(ag, dtype, kname, N, D):
    k = KERNELS[kname](ag, D)
    ko = oracle_of(ag, k, D)
    X, y, X64 = data(N, D, dtype)
    s2 = 0.05
    el = TOL[dtype]["el"]
    f = ag.GP(k)
    # Gram: symmetric with noise, and cross
    Kd = ag.cov(f(ag.RowVecs(X), s2))
    Ko = cr.kernelmatrix(ko, X64) + s2 * np.eye(N)
    np.testing.assert_allclose(Kd, Ko, rtol=el, atol=el)
    Xz, _, Xz64 = data(37, D, dtype, seed=5, dup=False)
    np.testing.assert_allclose(ag.kernelmatrix(k, ag.RowVecs(X), ag.RowVecs(Xz)), cr.kernelmatrix(ko, X64, Xz64), rtol=el, atol=el)
    np.testing.assert_allclose(ag.var(f, ag.RowVecs(Xz)), cr.kernelmatrix_diag(ko, Xz64), rtol=el, atol=el)
    # fit: logpdf for several right-hand sides, alpha
    Y = np.stack([y, y[::-1], 0.5 * y + 1], 1).astype(dtype)
    noise, mean = ref.NoiseSpec(0, s2), ref.MeanSpec()
    lp = ag.logpdf(f(ag.RowVecs(X), s2), Y)
    lp_o = cr.logpdf(ko, mean, noise, X64, Y.astype(np.float64))
    np.testing.assert_allclose(lp, lp_o, rtol=TOL[dtype]["rtol"], atol=0 if dtype == np.float64 else 1e-2)
    post = ag.posterior(f(ag.RowVecs(X), s2), y)
    po = cr.posterior(ko, mean, noise, X64, y.astype(np.float64))
    sc = np.abs(po["alpha"]).max()
    np.testing.assert_allclose(post.data.alpha, po["alpha"], rtol=1e-6 if dtype == np.float64 else 2e-2,
                               atol=(1e-7 if dtype == np.float64 else 1e-2) * sc)
    # predictions over the posterior
    m, v = ag.mean_and_var(post(ag.RowVecs(Xz), 0.01))
    mo, vo = cr.post_mean_and_var(po, Xz64, ref.NoiseSpec(0, 0.01))
    np.testing.assert_allclose(m, mo, rtol=el * 10, atol=el * 10)
    np.testing.assert_allclose(v, vo, rtol=el * 10, atol=el * 10)
    mc, Cc = ag.mean_and_cov(post(ag.RowVecs(Xz)))
    mco, Cco = cr.post_mean_and_cov(po, Xz64)
    np.testing.assert_allclose(Cc, Cco, rtol=el * 10, atol=el * 10)
    Yz = np.stack([mo + 0.1, mo - 0.2], 1).astype(dtype)
    lpz = ag.logpdf(post(ag.RowVecs(Xz), 0.05), Yz)
    np.testing.assert_allclose(lpz, cr.post_logpdf(po, Xz64, ref.NoiseSpec(0, 0.05), Yz.astype(np.float64)),
                               rtol=TOL[dtype]["rtol"] * 10, atol=0 if dtype == np.float64 else 1e-2)
    Z = np.random.default_rng(3).standard_normal((37, 2)).astype(dtype)
    smp = ag.rand_from_normals(post(ag.RowVecs(Xz), 0.05), Z)
    np.testing.assert_allclose(smp, cr.post_rand_from_Z(po, Xz64, ref.NoiseSpec(0, 0.05), Z.astype(np.float64)),
                               rtol=el * 10, atol=el * 10)
    # sequential conditioning
    X2, y2, X264 = data(29, D, dtype, seed=11, dup=False)
    p2 = ag.posterior(post(ag.RowVecs(X2), s2), y2)
    po2 = cr.posterior_sequential(po, ref.NoiseSpec(0, s2), X264, y2.astype(np.float64))
    m2, v2 = ag.mean_and_var(p2(ag.RowVecs(Xz)))
    m2o, v2o = cr.post_mean_and_var(po2, Xz64)
    np.testing.assert_allclose(m2, m2o, rtol=el * 10, atol=el * 10)
    np.testing.assert_allclose(v2, v2o, rtol=el * 10, atol=el * 10)


@pytest.mark.parametrize("dtype,N", [(np.float64, 8320), (np.float32, 4224)])
def test_composite_fit_on_int8_slice_cholesky(ag, dtype, N):
    """large enough for the automatic engine choice to take the int8-slice trailing update"""
    D = 1
    k = k_stationary(ag, D)
    ko = oracle_of(ag, k, D)
    X, y, X64 = data(N, D, dtype)
    s2 = 0.05
    lp = ag.logpdf(ag.GP(k)(ag.RowVecs(X), s2), y)
    Kc = np.empty((N, N))
    for i in range(0, N, 1024):  # the model's pairwise differences, in row blocks
        Kc[i:i + 1024] = cr.kernelmatrix(ko, X64[i:i + 1024], X64)
    Kc[np.diag_indices(N)] += s2
    U = ref.cholesky_upper(Kc)
    lp_o = -0.5 * (N * ref.LOG2PI + ref.logdet_chol(U) + ref.tr_Xt_invA_X(U, y.astype(np.float64)))
    assert abs(lp - lp_o) <= TOL[dtype]["rtol"] * abs(lp_o), (lp, lp_o)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname,D", [("stationary", 1), ("ard", 3), ("ard", 40), ("mixed", 3)])
def test_composite_logpdf_grad(ag, dtype, kname, D):
    k = KERNELS[kname](ag, D)
    ko = oracle_of(ag, k, D)
    N = 300
    X, y, X64 = data(N, D, dtype)
    s2 = np.random.default_rng(4).uniform(0.05, 0.1, N).astype(dtype)
    f = ag.GP(0.4, k)
    lp, g = ag.logpdf_grad(f(ag.RowVecs(X), s2), y)
    eng = ag.engine()
    post = ag.posterior(f(ag.RowVecs(X), s2), y)
    gd = np.zeros(int(eng.L.agp_post_grad_len(post.data.C.h)))
    eng.check(eng.L.agp_post_logpdf_grad(post.data.C.h, gd.ctypes.data_as(C.POINTER(C.c_double)), None))
    go, gno = cr.logpdf_grad(ko, ref.MeanSpec(1, 0.4), ref.NoiseSpec(1, v=s2.astype(np.float64)), X64, y.astype(np.float64))
    rt = 1e-7 if dtype == np.float64 else 2e-2
    scale = np.abs(go).max()
    np.testing.assert_allclose(gd, go, rtol=rt, atol=rt * scale)
    np.testing.assert_allclose(g["noise"], gno, rtol=rt, atol=rt * np.abs(gno).max())
    assert np.isclose(g["mean_c"], go[4], rtol=rt)
    # the per-parameter gradient is the descriptor's mapped back onto kernel_params(k)
    assert len(g["kernel"]) == len(ag.kernel_params(k))


def _co2():
    d = np.genfromtxt(os.path.join(ROOT, "tests", "golden", "CO2_data.csv"), delimiter=",")
    d = d[~np.isnan(d).any(1)]
    return d[:, 0], d[:, 1]


def _mauna_loa_kernel(ag, th):
    """build_gp_prior(theta) of examples/1-mauna-loa/script.jl:102-116, theta = log-parameters (period fixed at 1)"""
    e = np.exp(th)
    SE = lambda s, l: s ** 2 * ag.with_lengthscale(ag.SqExponentialKernel(), l)  # noqa: E731
    per = ag.with_lengthscale(ag.PeriodicKernel(r=[e[2] / 2]), 1.0)
    RQ = e[5] ** 2 * ag.with_lengthscale(ag.RationalQuadraticKernel(alpha=e[7]), e[6])
    return (SE(e[0], e[1]) + per * SE(e[3], e[4]) + RQ + (SE(e[8], e[9]) + e[10] ** 2 * ag.WhiteKernel()))


def _chain_log(ag, k, th, gk):
    """d loss / d log-theta from d logpdf / d kernel_params (kernel_params order: se_long s2, s | per s, r | se s2, s |
    rq s2, s, alpha | se s2, s | white s2)"""
    e = np.exp(th)
    p = ag.kernel_params(k)
    g = [float(np.sum(x)) for x in gk]
    # parameter -> (index in theta, d param / d log theta)
    dl = np.zeros(11)
    m = [(0, 2 * e[0] ** 2), (1, -p[1]), (None, 0), (2, p[3][0]), (3, 2 * e[3] ** 2), (4, -p[5]), (5, 2 * e[5] ** 2),
         (6, -p[7]), (7, e[7]), (8, 2 * e[8] ** 2), (9, -p[10]), (10, 2 * e[10] ** 2)]
    for (i, dp), gi in zip(m, g):
        if i is not None:
            dl[i] += gi * dp
    return -dl


def test_mauna_loa_replay(ag):
    """examples/1-mauna-loa: the prior, f(xtrain) with the default 1e-18 noise, logpdf and its gradient at theta_init
    against the model, then L-BFGS-B on the device's loss and gradient; at the optimum the model agrees"""
    from scipy.optimize import minimize
    x, y = _co2()
    tr = x < 2004
    xtr, ytr, xte = x[tr], y[tr], x[~tr][:50]
    th0 = np.array([4.0, 4.0, 0.0, 1.0, 4.0, 0.0, 0.0, -1.0, -2.0, -2.0, -2.0])
    X = xtr[:, None]

    def dev(th):
        k = _mauna_loa_kernel(ag, th)
        lp, g = ag.logpdf_grad(ag.GP(k)(xtr), ytr)
        return -lp, _chain_log(ag, k, th, g["kernel"]), k

    def loss(th):  # a trial step whose covariance is not positive definite is a step the line search must shorten
        try:
            return dev(th)[:2]
        except ag.PosDefException:
            return 1e30, np.zeros_like(th)

    def model(th):
        k = _mauna_loa_kernel(ag, th)
        ko = oracle_of(ag, k, 1)
        go, _ = cr.logpdf_grad(ko, ref.MeanSpec(), ref.NoiseSpec(0, 1e-18), X, ytr)
        lp = cr.logpdf(ko, ref.MeanSpec(), ref.NoiseSpec(0, 1e-18), X, ytr)
        keep = []
        fl = ag.api._Flat(k, 1)
        fl.struct(np.float64, keep)
        return -lp, _chain_log(ag, k, th, fl.params_grad(go)), ko

    l0, g0, _ = dev(th0)
    lo0, go0, _ = model(th0)
    assert abs(l0 - lo0) <= 1e-8 * abs(lo0)
    np.testing.assert_allclose(g0, go0, rtol=1e-6, atol=1e-6 * np.abs(go0).max())
    res = minimize(loss, th0, jac=True, method="L-BFGS-B", bounds=[(t - 4, t + 4) for t in th0], options=dict(maxiter=200))
    lo, go, ko = model(res.x)
    # the optimum drives the white-noise variance down, so the covariance there is far worse conditioned than at
    # theta_init: two fp64 factorisations of it (device and model) agree to a few 1e-8 of the loss, not 1e-8.  The device
    # gradient's fp64 atomics make the L-BFGS path, and so the optimum reached, vary slightly from run to run.
    assert abs(res.fun - lo) <= 3e-8 * abs(lo)
    assert res.fun < l0
    assert np.linalg.norm(go) <= 1e-2 * max(1.0, np.linalg.norm(go0)), (np.linalg.norm(go), res.message)
    k = _mauna_loa_kernel(ag, res.x)
    post = ag.posterior(ag.GP(k)(xtr), ytr)
    m, v = ag.mean_and_var(post(xte))
    po = cr.posterior(ko, ref.MeanSpec(), ref.NoiseSpec(0, 1e-18), X, ytr)
    mo, vo = cr.post_mean_and_var(po, xte[:, None])
    np.testing.assert_allclose(m, mo, rtol=1e-7, atol=1e-6)
    np.testing.assert_allclose(v, vo, rtol=1e-5, atol=1e-6)


def test_composite_rejections(ag):
    cabi = ag._cabi
    eng = ag.engine()
    k = k_stationary(ag, 1)
    x = np.linspace(0, 1, 20)
    f = ag.GP(k)
    with pytest.raises(ag.AGPError) as e:
        ag.approx_log_evidence(ag.VFE(f(x[:5])), f(x, 0.1), np.sin(x))
    assert e.value.code == cabi.AGP_ERR_UNSUPPORTED and "VFE" in str(e.value)
    # a factor-only family at top level of agp_kernel
    ks = cabi.agp_kernel()
    ks.family, ks.variance, ks.scale = cabi.AGP_RQ, 1.0, 1.0
    X = np.ascontiguousarray(x[:, None])
    K = np.empty((20, 20), order="F")
    rc = eng.L.agp_gram(eng.h, cabi.AGP_F64, C.byref(ks), 0, cabi.ptr(X), 20, 1, None, 0, None, cabi.ptr(K))
    assert rc == cabi.AGP_ERR_UNSUPPORTED
    # invalid descriptors
    keep = []
    kc = ag.api._Flat(ag.RationalQuadraticKernel(alpha=-1.0) + ag.SqExponentialKernel(), 1).struct(np.float64, keep)
    rc = eng.L.agp_gram(eng.h, cabi.AGP_F64, C.byref(kc), 0, cabi.ptr(X), 20, 1, None, 0, None, cabi.ptr(K))
    assert rc == cabi.AGP_ERR_INVALID and b"alpha" in eng.L.agp_last_error(eng.h)
    kc.composite.contents.nterms = 9
    rc = eng.L.agp_gram(eng.h, cabi.AGP_F64, C.byref(kc), 0, cabi.ptr(X), 20, 1, None, 0, None, cabi.ptr(K))
    assert rc == cabi.AGP_ERR_INVALID

    def gram_rc(kc):
        return eng.L.agp_gram(eng.h, cabi.AGP_F64, C.byref(kc), 0, cabi.ptr(X), 20, 1, None, 0, None, cabi.ptr(K))
    # a top-level transform on a composite (here ARD without weights) is declined before any upload or launch
    kc = ag.api._Flat(k, 1).struct(np.float64, keep)
    kc.transform, kc.ard = 2, None
    assert gram_rc(kc) == cabi.AGP_ERR_INVALID
    lp = np.empty(1)
    Y = np.sin(X[:, 0]).copy()
    rc = eng.L.agp_fit(eng.h, cabi.AGP_F64, C.byref(kc), None, None, 0, cabi.ptr(X), 20, 1, cabi.ptr(Y), 1, cabi.ptr(lp), None, None)
    assert rc == cabi.AGP_ERR_INVALID
    # a factor with an ARD transform but no weights
    kc = ag.api._Flat(ag.SqExponentialKernel().compose(ag.ARDTransform([0.5])) + ag.WhiteKernel(), 1).struct(np.float64, keep)
    kc.composite.contents.factors[0].ard = None
    assert gram_rc(kc) == cabi.AGP_ERR_INVALID and b"ARD" in eng.L.agp_last_error(eng.h)
    # Periodic r <= 0
    kc = ag.api._Flat(ag.PeriodicKernel(r=[-1.0]) + ag.SqExponentialKernel(), 1).struct(np.float64, keep)
    assert gram_rc(kc) == cabi.AGP_ERR_INVALID and b"r must be > 0" in eng.L.agp_last_error(eng.h)
    kc = ag.api._Flat(ag.PeriodicKernel(r=[0.0]) * ag.SqExponentialKernel(), 1).struct(np.float64, keep)
    assert gram_rc(kc) == cabi.AGP_ERR_INVALID
    # the engine still works after the rejections
    np.testing.assert_allclose(ag.kernelmatrix(k, x), cr.kernelmatrix(oracle_of(ag, k, 1), X), rtol=1e-12, atol=1e-12)


def test_composite_rejected_on_distributed_context(ag):
    """a distributed (NCCL) context declines composite kernels; a one-rank communicator is enough to reach that path"""
    cabi = ag._cabi
    L = cabi.lib()
    idbuf = np.zeros(128, dtype=np.uint8)
    assert L.agp_nccl_unique_id(idbuf.ctypes.data) == 0
    h = C.c_void_p()
    assert L.agp_init_dist(C.byref(h), 0, 0, 1, 1, 1, idbuf.ctypes.data, None) == 0
    try:
        keep = []
        kc = ag.api._Flat(k_stationary(ag, 1), 1).struct(np.float64, keep)
        X = np.ascontiguousarray(np.linspace(0, 1, 40)[:, None])
        Y = np.sin(X[:, 0]).copy()
        lp = np.empty(1)
        rc = L.agp_fit(h, cabi.AGP_F64, C.byref(kc), None, None, 0, cabi.ptr(X), 40, 1, cabi.ptr(Y), 1, cabi.ptr(lp), None, None)
        assert rc == cabi.AGP_ERR_UNSUPPORTED
        assert b"single-GPU" in L.agp_last_error(h)
    finally:
        L.agp_destroy(h)

