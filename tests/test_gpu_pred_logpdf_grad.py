"""The gradient of the held-out log-likelihood logpdf(posterior(fx, y)(x*, Sigma*), Y*) on the device
(agp_post_pred_logpdf_grad), in fp64 and fp32: against the CPU model tests/pred_logpdf_grad_ref.py for the five
single-kernel families under every transform in the row, column and vector containers, per-point noises and vector means,
composites and the Mauna Loa kernel on a train / held-out split of the CO2 data; S = 1 against S columns with weights e_s;
central differences of agp_post_logpdf over refits; the int8-slice and tensor forward-substitution sizes with the branch
asserted from the launch counter; device memory, determinism, the error codes; and a short L-BFGS-B replay of
validation-likelihood training against the model's path.
Tolerances: rtol 1e-7 (fp64) / 2e-2 (fp32, against the model on the fp32-rounded inputs), atol the same times max|g|."""
import ctypes as C

import numpy as np
import pytest

import composite_ref as cr
import pred_logpdf_grad_ref as pr
from oracle import agp_ref as ref
from test_gpu_composite import KERNELS, _co2, _mauna_loa_kernel, oracle_of
from test_gpu_rand_grad import _DevArr, _launches, check_single, close, container, kernel, x_rows

pytestmark = pytest.mark.gpu
RT = {np.float64: 1e-7, np.float32: 2e-2}
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]


def data(N, M, D, S, dtype, seed=0):
    rng = np.random.default_rng(seed + 7 * N + 3 * M + D + 5 * S)
    return (rng.uniform(-2, 2, (N, D)).astype(dtype), rng.standard_normal(N).astype(dtype),
            rng.uniform(-2.2, 2.2, (M, D)).astype(dtype), rng.standard_normal((M, S)).astype(dtype))


def weights(S, kind):
    if kind is None:
        return None
    w = np.random.default_rng(S).uniform(-1.5, 2.0, S)
    w[S // 2] = 0.0
    return w


def f64(*a):
    return [np.asarray(v, dtype=np.float64) for v in a]


def check_all(g, want, spec, kind, rt, kernel=True):
    if kernel:
        check_single(g, want, spec, rt)
    close(g["noise"], want["grad"][3], rt)
    close(g["mean_c"], want["grad"][4], rt)
    close(g["noise_s"], np.sum(want["noise_s_diag"]), rt)
    close(g["y"], want["y"], rt)
    close(g["Y"], want["Ys"], rt)
    close(x_rows(g["x"], kind), want["x"], rt)
    close(x_rows(g["xs"], kind), want["xs"], rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_matches_model(ag, family, transform, dtype):
    rt = RT[dtype]
    for N, M, D, S, kind, wkind in [(1, 1, 1, 1, "vec", None), (63, 17, 3, 2, "row", "mixed"), (333, 129, 1, 3, "col", None),
                                    (333, 200, 40, 2, "row", "mixed"), (1300, 1000, 3, 130, "col", "mixed")]:
        k, spec = kernel(ag, family, transform, D)
        X, y, Xs, Ys = data(N, M, D, S, dtype)
        w = weights(S, wkind)
        p = ag.posterior(ag.GP(0.3, k)(container(ag, X, kind), 0.1), y)
        lp, g = ag.posterior_logpdf_grad(p(container(ag, Xs, kind), 0.05), Ys, lp_bar=w, inputs=True)
        want = pr.pred_logpdf_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs),
                                   ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.05), *f64(Ys), w)
        assert g["xs"].dtype == dtype and g["Y"].dtype == dtype and g["Y"].shape == (M, S)
        # fp32 Linear kernel gradients are measured at 3e-3 .. 0.43 off the model (DESIGN s6,
        # tools/pred_logpdf_grad_fp32_error.py; up to 0.4 on this grid's Scale / ARD cases): the posterior covariance of a
        # rank-D prior is the test noise plus O(D / N), so they are differences of nearly equal terms.  Held to the model
        # in fp64 only; every other fp32 output is held to 2e-2
        linear32 = spec.family == cr.LINEAR and dtype == np.float32
        check_all(g, want, spec, kind, rt, kernel=not linear32)
        close(lp, want["lp"], 10 * rt)
        close(lp, ag.logpdf(p(container(ag, Xs, kind), 0.05), Ys), 10 * rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_per_point_noises_and_vector_means(ag, dtype):
    N, M, D, S = 500, 300, 2, 5
    k, spec = kernel(ag, cr.MATERN32, cr.T_ARD, D)
    X, y, Xs, Ys = data(N, M, D, S, dtype, seed=2)
    rng = np.random.default_rng(2)
    s2, s2s = rng.uniform(0.05, 0.2, N), rng.uniform(0.02, 0.1, M)
    w = weights(S, "mixed")
    p = ag.posterior(ag.GP(ag.CustomMean(lambda x: np.sin(x[0])), k)(ag.RowVecs(X), s2), y)
    lp, g = ag.posterior_logpdf_grad(p(ag.RowVecs(Xs), s2s), Ys, lp_bar=w, inputs=True)
    r = lambda a: np.asarray(a).astype(dtype).astype(np.float64)  # noqa: E731
    X64, Xs64 = f64(X, Xs)
    want = pr.pred_logpdf_grad(spec, ref.MeanSpec(2, v=r(np.sin(X64[:, 0]))), ref.NoiseSpec(1, v=r(s2)), X64, *f64(y), Xs64,
                               ref.MeanSpec(2, v=r(np.sin(Xs64[:, 0]))), ref.NoiseSpec(1, v=r(s2s)), *f64(Ys), w)
    rt = RT[dtype]
    for key, wk in [("noise", "noise_diag"), ("mean_v", "mean_diag"), ("noise_s", "noise_s_diag"),
                    ("mean_s_v", "mean_s_diag"), ("x", "x"), ("xs", "xs"), ("y", "y"), ("Y", "Ys")]:
        close(g[key], want[wk], rt)
    check_single(g, want, spec, rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname,D", [("stationary", 1), ("ard", 3), ("mixed", 3)])
def test_composite(ag, dtype, kname, D):
    k = KERNELS[kname](ag, D)
    ko = oracle_of(ag, k, D)
    X, y, Xs, Ys = data(333, 150, D, 3, dtype, seed=6)
    w = weights(3, "mixed")
    p = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    lp, g = ag.posterior_logpdf_grad(p(ag.RowVecs(Xs), 0.05), Ys, lp_bar=w, inputs=True)
    want = pr.pred_logpdf_grad(ko, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs), ref.MeanSpec(1, 0.3),
                               ref.NoiseSpec(0, 0.05), *f64(Ys), w)
    rt = RT[dtype]
    wk = ag.api._Flat(k, D).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(v, dtype=np.float64)).max() for v in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(np.asarray(a, dtype=np.float64), b, rtol=rt, atol=rt * scale)
    for key, wkey in [("x", "x"), ("xs", "xs"), ("y", "y"), ("Y", "Ys")]:
        close(g[key], want[wkey], rt)
    close(g["noise"], want["grad"][3], rt)
    close(g["mean_c"], want["grad"][4], rt)


def test_mauna_loa_held_out(ag):
    """the Mauna Loa kernel on the CO2 data: train on the first 400 months, score the next 150"""
    x, y = _co2()
    xtr, ytr, xte, yte = x[:400], y[:400], x[400:550], y[400:550]
    k = _mauna_loa_kernel(ag, np.array([4.0, 4.0, 0.0, 1.0, 4.0, 0.0, 0.0, -1.0, -2.0, -2.0, -2.0]))
    ko = oracle_of(ag, k, 1)
    m = float(np.mean(ytr))
    p = ag.posterior(ag.GP(m, k)(xtr, 0.05), ytr)
    lp, g = ag.posterior_logpdf_grad(p(xte, 0.05), yte, inputs=True)
    want = pr.pred_logpdf_grad(ko, ref.MeanSpec(1, m), ref.NoiseSpec(0, 0.05), xtr[:, None], ytr, xte[:, None], ref.MeanSpec(1, m),
                               ref.NoiseSpec(0, 0.05), yte)
    wk = ag.api._Flat(k, 1).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(v, dtype=np.float64)).max() for v in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(a, b, rtol=1e-7, atol=1e-7 * scale)
    close(lp, want["lp"][0], 1e-9)
    close(g["x"], want["x"][:, 0], 1e-7)
    close(g["xs"], want["xs"][:, 0], 1e-7)
    close(g["noise"], want["grad"][3], 1e-7)
    close(g["noise_s"], np.sum(want["noise_s_diag"]), 1e-7)
    close(g["mean_c"], want["grad"][4], 1e-7)
    close(g["y"], want["y"], 1e-7)
    close(g["Y"], want["Ys"][:, 0], 1e-7)


# ---- the raw entry point on a handle -----------------------------------------------------------------------------------
def _call(ag, h, Xs, Ys, S=None, w=None, outs=None, layout=0, mean=None, noise=None, M=None):
    cabi = ag._cabi
    eng = ag.engine()
    p = lambda a: a if isinstance(a, int) else cabi.ptr(a)  # noqa: E731
    dp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    o = outs or {}
    M = (Xs.shape[0] if layout == 0 else Xs.shape[-1]) if M is None else M
    return eng.L.agp_post_pred_logpdf_grad(
        h, layout, p(Xs), M, None if mean is None else C.byref(mean), None if noise is None else C.byref(noise), p(Ys),
        (Ys.shape[1] if Ys is not None else 1) if S is None else S, dp(w), p(o.get("lp")), dp(o.get("g")), p(o.get("nd")),
        p(o.get("md")), p(o.get("yb")), p(o.get("xg")), p(o.get("nsd")), p(o.get("msd")), p(o.get("ysb")), p(o.get("xsg")))


def _outs(N, M, D, S, dtype, glen=None):
    e = lambda *s: np.empty(s, dtype=dtype, order="F")  # noqa: E731
    # the input gradients point-major: D x n column-major, i.e. n x D row-major
    return dict(lp=e(S), g=np.zeros(5 + D if glen is None else glen), nd=e(N), md=e(N), yb=e(N),
                xg=np.empty((N, D), dtype=dtype), nsd=e(M), msd=e(M), ysb=e(M, S), xsg=np.empty((M, D), dtype=dtype))


def _noise(ag, s):
    return ag._cabi.agp_noise(0, s, None)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_unit_weights_match_single_columns(ag, dtype):
    """S columns with w = e_s equal the call on column s alone, in every output"""
    N, M, D, S = 600, 250, 3, 4
    k, _ = kernel(ag, cr.MATERN12, cr.T_ARD, D)
    X, y, Xs, Ys = data(N, M, D, S, dtype, seed=5)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Yf, Xsc = post.data.C.h, np.asfortranarray(Ys), np.ascontiguousarray(Xs)
    for s in (0, 2, 3):
        e = np.zeros(S)
        e[s] = 1.0
        a, b = _outs(N, M, D, S, dtype), _outs(N, M, D, 1, dtype)
        assert _call(ag, h, Xsc, Yf, w=e, outs=a, noise=_noise(ag, 0.05)) == 0
        assert _call(ag, h, Xsc, np.asfortranarray(Ys[:, s:s + 1]), outs=b, noise=_noise(ag, 0.05)) == 0
        rt = 1e-10 if dtype == np.float64 else 1e-4
        for key in ("g", "nd", "md", "yb", "xg", "nsd", "msd", "xsg"):
            close(a[key], b[key], rt)
        close(a["ysb"][:, s], b["ysb"][:, 0], rt)
        assert np.all(a["ysb"][:, [j for j in range(S) if j != s]] == 0.0)
        close(a["lp"][s], b["lp"][0], rt)


def test_central_differences_over_refits(ag):
    """the kernel scale, the training noise, an input, a target and a test input against central differences of
    agp_post_logpdf over refits"""
    N, M, D = 120, 40, 2
    X, y, Xs, Ys = data(N, M, D, 1, np.float64, seed=11)
    ls, s2 = 0.9, 0.1

    def F(ls_=ls, s2_=s2, X_=X, y_=y, Xs_=Xs):
        k = ag.with_lengthscale(ag.Matern52Kernel(), ls_)
        p = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X_), s2_), y_)
        return float(ag.logpdf(p(ag.RowVecs(Xs_), 0.05), Ys[:, 0]))
    p = ag.posterior(ag.GP(0.3, ag.with_lengthscale(ag.Matern52Kernel(), ls))(ag.RowVecs(X), s2), y)
    lp, g = ag.posterior_logpdf_grad(p(ag.RowVecs(Xs), 0.05), Ys[:, 0], inputs=True)
    h = 1e-5
    fd = lambda a, b: (a - b) / (2 * h)  # noqa: E731
    s = 1.0 / ls  # the Scale transform's s
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
        Xsp, Xsm = Xs.copy(), Xs.copy()
        Xsp[i % M, d] += h
        Xsm[i % M, d] -= h
        v = fd(F(Xs_=Xsp), F(Xs_=Xsm))
        assert abs(g["xs"][i % M, d] - v) <= 1e-6 * max(1.0, abs(v)), (i, d, g["xs"][i % M, d], v)
    yp, ym = y.copy(), y.copy()
    yp[10] += h
    ym[10] -= h
    v = fd(F(y_=yp), F(y_=ym))
    assert abs(g["y"][10] - v) <= 1e-6 * max(1.0, abs(v)), (g["y"][10], v)


def _tensor_case(ag, dtype, N, M, key, mode):
    """the fit and the call under `key` = mode, and again under 0 (the tile kernels): the launch counts of the two calls
    differ, and both agree with the model"""
    eng = ag.engine()
    D, S = 2, 2
    k, spec = kernel(ag, cr.SE, cr.T_ARD, D)
    X, y, Xs, Ys = data(N, M, D, S, dtype, seed=12)
    Yf, Xsc, w = np.asfortranarray(Ys), np.ascontiguousarray(Xs), np.array([0.7, -1.3])
    cfg = eng.get_config()
    res = []
    try:
        for m in (mode, 0):
            eng.set_config(**{key: m})  # before the fit: the handle's own factor comes from this policy too
            post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
            o = _outs(N, M, D, S, dtype)
            n, rc = _launches(ag, lambda: _call(ag, post.data.C.h, Xsc, Yf, w=w, outs=o, noise=_noise(ag, 0.05)))
            assert rc == 0
            res.append((n, o))
    finally:
        eng.set_config(**{key: getattr(cfg, key)})
    assert res[0][0] != res[1][0], (res[0][0], res[1][0])
    want = pr.pred_logpdf_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs), ref.MeanSpec(1, 0.3),
                               ref.NoiseSpec(0, 0.05), *f64(Ys), w)
    rt = RT[dtype]
    for _, o in res:
        for key_, wk in [("nd", "noise_diag"), ("yb", "y"), ("xg", "x"), ("nsd", "noise_s_diag"), ("msd", "mean_s_diag"),
                         ("ysb", "Ys"), ("xsg", "xs"), ("lp", "lp")]:
            close(o[key_], want[wk], rt)
        close(o["g"][[0, 3, 4, 5, 6]], want["grad"][[0, 3, 4, 5, 6]], rt)


def test_int8_slice_forced_fp64(ag):
    """fp64 at N = 2304 with the int8-slice kernels forced (fp64_mode = 1) for the fit and the call: the handle's factor,
    the factor of Sigma (M = 512) and the tensor forward substitution of K_xs"""
    _tensor_case(ag, np.float64, 2304, 512, "fp64_mode", 1)


@pytest.mark.parametrize("dtype,N,key", [(np.float64, 8320, "fp64_mode"), (np.float32, 4224, "fp32_mode")])
def test_int8_slice_automatic(ag, dtype, N, key):
    """fp64 N = 8320 and fp32 N = 4224: the automatic policy (-1) takes the int8-slice kernels"""
    _tensor_case(ag, dtype, N, 600, key, -1)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_determinism_null_outputs_and_layouts(ag, dtype):
    N, M, D, S = 700, 300, 3, 1100
    k, _ = kernel(ag, cr.MATERN32, cr.T_SCALE, D)
    X, y, Xs, Ys = data(N, M, D, S, dtype, seed=7)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Yf, Xsc, w = post.data.C.h, np.asfortranarray(Ys), np.ascontiguousarray(Xs), weights(S, "mixed")
    outs = []
    for _ in range(2):
        o = _outs(N, M, D, S, dtype)
        assert _call(ag, h, Xsc, Yf, w=w, outs=o, noise=_noise(ag, 0.05)) == 0
        outs.append(o)
    for key in outs[0]:
        if key != "g":
            assert outs[0][key].tobytes() == outs[1][key].tobytes(), key
    assert outs[0]["g"][3:5].tobytes() == outs[1]["g"][3:5].tobytes()
    np.testing.assert_allclose(outs[0]["g"], outs[1]["g"], rtol=1e-10, atol=1e-10 * np.abs(outs[0]["g"]).max())
    for key in ("ysb", "msd", "lp", "yb", "xsg"):  # each alone: the rest of the work is skipped, the bits are the same
        o = {key: np.empty_like(outs[0][key])}
        assert _call(ag, h, Xsc, Yf, w=w, outs=o, noise=_noise(ag, 0.05)) == 0
        assert o[key].tobytes() == outs[0][key].tobytes(), key
    # feature-major: the input points and both input gradients as M x D / N x D column-major
    o = dict(xg=np.empty((N, D), dtype=dtype, order="F"), xsg=np.empty((M, D), dtype=dtype, order="F"))
    assert _call(ag, h, np.asfortranarray(Xs), Yf, w=w, outs=o, layout=1, M=M, noise=_noise(ag, 0.05)) == 0
    assert o["xg"].tobytes(order="F") == np.asfortranarray(outs[0]["xg"]).tobytes(order="F")
    assert o["xsg"].tobytes(order="F") == np.asfortranarray(outs[0]["xsg"]).tobytes(order="F")
    assert _call(ag, h, Xsc, Yf, w=w) == 0  # nothing requested


def test_device_memory(ag):
    torch = pytest.importorskip("torch")
    cabi = ag._cabi
    eng = ag.engine()
    N, M, D, S = 500, 200, 4, 130
    k, _ = kernel(ag, cr.SE, cr.T_ARD, D)
    X, y, Xs, Ys = data(N, M, D, S, np.float64, seed=8)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Yf, Xsc, w = post.data.C.h, np.asfortranarray(Ys), np.ascontiguousarray(Xs), weights(S, "mixed")
    o0 = _outs(N, M, D, S, np.float64)
    assert _call(ag, h, Xsc, Yf, w=w, outs=o0, noise=_noise(ag, 0.05)) == 0
    Yd = torch.from_numpy(Yf.ravel(order="F").copy()).cuda()
    Xd = torch.from_numpy(Xsc.ravel().copy()).cuda()
    dev = {key: torch.empty(v.size, dtype=torch.float64, device="cuda") for key, v in o0.items() if key != "g"}
    o = {key: t.data_ptr() for key, t in dev.items()}
    o["g"] = np.zeros(5 + D)
    torch.cuda.synchronize()
    eng.set_memspace(cabi.AGP_MEM_DEVICE)
    try:
        rc = _call(ag, h, _DevArr(Xd, M, D), _DevArr(Yd, M, S), w=w, outs=o, M=M, noise=_noise(ag, 0.05))
    finally:
        eng.set_memspace(cabi.AGP_MEM_HOST)
    assert rc == 0
    for key, t in dev.items():
        assert t.cpu().numpy().tobytes() == o0[key].tobytes(order="A"), key
    np.testing.assert_allclose(o["g"], o0["g"], rtol=1e-10, atol=1e-10 * np.abs(o0["g"]).max())


def test_errors(ag):
    cabi = ag._cabi
    N, M, D, S = 50, 20, 2, 3
    k, _ = kernel(ag, cr.SE, cr.T_SCALE, D)
    X, y, Xs, Ys = data(N, M, D, S, np.float64, seed=9)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Yf, Xsc = post.data.C.h, np.asfortranarray(Ys), np.ascontiguousarray(Xs)
    g = dict(g=np.zeros(5 + D))
    assert _call(ag, h, Xsc, Yf, outs=g, S=0) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Yf, outs=g, S=-2) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, None, outs=g) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Yf, outs=g, layout=2) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Yf, outs=g, mean=cabi.agp_mean(2, 0.0, None)) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Yf, outs=g, noise=cabi.agp_noise(1, 0.0, None)) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Yf, outs=g, M=0) == cabi.AGP_ERR_DIM_MISMATCH
    # a test covariance that is not positive definite: a negative test noise larger than the posterior variance
    assert _call(ag, h, Xsc, Yf, outs=g, noise=_noise(ag, -5.0)) == cabi.AGP_ERR_NOT_POSDEF
    assert ag.engine().L.agp_post_pred_logpdf_grad(None, 0, cabi.ptr(Xsc), M, None, None, cabi.ptr(Yf), S, *([None] * 11)) == \
        cabi.AGP_ERR_INVALID
    X2, y2, _, _ = data(20, 1, D, 1, np.float64, seed=10)
    post2 = ag.posterior(post(ag.RowVecs(X2), 0.1), y2)
    assert _call(ag, post2.data.C.h, Xsc, Yf, outs=dict(g=np.zeros(5 + D))) == cabi.AGP_ERR_UNSUPPORTED
    o = _outs(N, M, D, S, np.float64)  # the handle still works after every refusal
    assert _call(ag, h, Xsc, Yf, outs=o) == 0
    assert np.all(np.isfinite(o["g"]))


def test_lbfgs_validation_training_replay(ag):
    """validation-likelihood training: L-BFGS-B over (log variance, log lengthscale, log noise) of an SE prior, maximising
    the held-out logpdf, with the device gradient and with the model's: the two paths agree"""
    from scipy.optimize import minimize
    N, M, D = 200, 80, 1
    X, y, Xs, Ys = data(N, M, D, 1, np.float64, seed=13)
    y = np.sin(2 * X[:, 0]) + 0.1 * y
    Ys = (np.sin(2 * Xs[:, 0]) + 0.1 * Ys[:, 0])

    def dev(th):
        v, ls, s2 = np.exp(th)
        k = v * ag.with_lengthscale(ag.SqExponentialKernel(), ls)
        p = ag.posterior(ag.GP(k)(X[:, 0], s2), y)
        lp, g = ag.posterior_logpdf_grad(p(Xs[:, 0], s2), Ys)
        # d/d log ls = -s d/ds (s = 1/ls); the noise is shared: both sides
        return -lp, -np.array([g["variance"] * v, -g["scale"] / ls, (g["noise"] + g["noise_s"]) * s2])

    def model(th):
        v, ls, s2 = np.exp(th)
        r = pr.pred_logpdf_grad(ref.KernelSpec(cr.SE, v, cr.T_SCALE, 1.0 / ls), ref.MeanSpec(), ref.NoiseSpec(0, s2), X, y, Xs,
                                ref.MeanSpec(), ref.NoiseSpec(0, s2), Ys)
        return -r["lp"][0], -np.array([r["grad"][0] * v, -r["grad"][1] / ls, (r["grad"][3] + np.sum(r["noise_s_diag"])) * s2])
    th0 = np.log([1.0, 0.5, 0.05])
    paths = []
    for fun in (dev, model):
        path = []
        res = minimize(fun, th0, jac=True, method="L-BFGS-B", callback=lambda t: path.append(t.copy()),
                       options=dict(maxiter=8))
        paths.append((np.array(path), res.fun))
    assert len(paths[0][0]) == len(paths[1][0]) > 2
    np.testing.assert_allclose(paths[0][0], paths[1][0], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(paths[0][1], paths[1][1], rtol=1e-8)
