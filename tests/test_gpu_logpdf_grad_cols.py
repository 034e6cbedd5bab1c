"""The gradient of sum_s w_s logpdf(fx, Y[:, s]) for a matrix Y on the device (agp_post_logpdf_grad_cols), in fp64 and fp32:
against the CPU model tests/logpdf_grad_cols_ref.py for the five single-kernel families under every transform in the row,
column and vector containers, S across the border width (128) and the 1024-column chunk, lp_bar NULL or mixed, a Y other
than the fitted one, composites and the Mauna Loa kernel on the CO2 data; against agp_post_logpdf_grad_x on the same handle
at S = 1 and, by linearity in w, on fits of single columns (also at the int8-slice sizes); device memory, determinism, the
error codes, and the reference's matrix logpdf gradient checks.
Tolerances: rtol 1e-7 (fp64) / 2e-2 (fp32, against the model on the fp32-rounded inputs), atol the same times max|g|."""
import ctypes as C

import numpy as np
import pytest

import composite_ref as cr
import logpdf_grad_cols_ref as lc
from oracle import agp_ref as ref
from test_gpu_composite import KERNELS, _co2, _mauna_loa_kernel, oracle_of
from test_gpu_rand_grad import _DevArr, _launches, check_single, close, container, kernel, x_rows

pytestmark = pytest.mark.gpu
RT = {np.float64: 1e-7, np.float32: 2e-2}
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]


def data(N, D, S, dtype, seed=0):
    rng = np.random.default_rng(seed + 7 * N + D + 3 * S)
    return rng.uniform(-2, 2, (N, D)).astype(dtype), rng.standard_normal((N, S)).astype(dtype)


def weights(S, kind):
    if kind is None:
        return None
    w = np.random.default_rng(S).uniform(-1.5, 2.0, S)
    w[S // 2] = 0.0
    return w


def check_all(g, want, spec, kind, rt):
    check_single(g, want, spec, rt)
    close(g["noise"], want["grad"][3], rt)
    close(g["mean_c"], want["grad"][4], rt)
    close(g["Y"], want["Y"], rt)
    close(x_rows(g["x"], kind), want["x"], rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_matches_model(ag, family, transform, dtype):
    rt = RT[dtype]
    for N, D, S, kind, wkind in [(1, 1, 1, "vec", None), (63, 3, 2, "row", "mixed"), (333, 1, 129, "col", None),
                                 (333, 3, 1500, "row", "mixed"), (333, 40, 2, "row", None), (1300, 3, 128, "col", "mixed")]:
        k, spec = kernel(ag, family, transform, D)
        X, Y = data(N, D, S, dtype)
        w = weights(S, wkind)
        lp, g = ag.loglikelihood_grad(ag.GP(0.3, k)(container(ag, X, kind), 0.1), Y, lp_bar=w, inputs=True)
        X64, Y64 = X.astype(np.float64), Y.astype(np.float64)
        want = lc.logpdf_grad_cols(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X64, Y64, w)
        assert g["x"].dtype == dtype and g["Y"].dtype == dtype and g["Y"].shape == (N, S)
        check_all(g, want, spec, kind, rt)
        close(lp, ref.logpdf(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X64, Y64), 10 * rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_wide_inputs(ag, dtype):
    N, D, S = 1300, 40, 129
    k, spec = kernel(ag, cr.SE, cr.T_ARD, D)
    X, Y = data(N, D, S, dtype, seed=1)
    lp, g = ag.loglikelihood_grad(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), Y, inputs=True)
    want = lc.logpdf_grad_cols(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X.astype(np.float64), Y.astype(np.float64))
    check_all(g, want, spec, "row", RT[dtype])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_per_point_noise_and_vector_mean(ag, dtype):
    N, D, S = 500, 2, 5
    k, spec = kernel(ag, cr.MATERN32, cr.T_ARD, D)
    X, Y = data(N, D, S, dtype, seed=2)
    s2 = np.random.default_rng(2).uniform(0.05, 0.2, N)
    w = weights(S, "mixed")
    lp, g = ag.loglikelihood_grad(ag.GP(ag.CustomMean(lambda x: np.sin(x[0])), k)(ag.RowVecs(X), s2), Y, lp_bar=w, inputs=True)
    X64 = X.astype(np.float64)
    mv = np.sin(X64[:, 0].astype(dtype).astype(np.float64))
    want = lc.logpdf_grad_cols(spec, ref.MeanSpec(2, v=mv), ref.NoiseSpec(1, v=s2.astype(dtype).astype(np.float64)), X64,
                               Y.astype(np.float64), w)
    rt = RT[dtype]
    close(g["noise"], want["noise_diag"], rt)
    close(g["mean_v"], want["mean_diag"], rt)
    close(g["x"], want["x"], rt)
    close(g["Y"], want["Y"], rt)
    check_single(g, want, spec, rt)


# ---- the raw entry point on a handle -----------------------------------------------------------------------------------
def _cols(ag, h, Y, S=None, w=None, g=None, nd=None, md=None, xg=None, yb=None, layout=0, mean=None):
    cabi = ag._cabi
    eng = ag.engine()
    p = lambda a: a if isinstance(a, int) else cabi.ptr(a)  # noqa: E731
    dp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    return eng.L.agp_post_logpdf_grad_cols(h, None if mean is None else C.byref(mean), p(Y),
                                           (Y.shape[1] if Y is not None else 1) if S is None else S, dp(w), dp(g), p(nd),
                                           p(md), layout, p(xg), p(yb))


def _grad_x(ag, h, N, D, dtype):
    eng = ag.engine()
    g, nd, xg = np.zeros(5 + D), np.empty(N, dtype=dtype), np.empty((N, D), dtype=dtype)
    assert eng.L.agp_post_logpdf_grad_x(h, g.ctypes.data_as(C.POINTER(C.c_double)), ag._cabi.ptr(nd), 0, ag._cabi.ptr(xg)) == 0
    return g, nd, xg


def _outs(N, D, S, dtype):
    return (np.zeros(5 + D), np.empty(N, dtype=dtype), np.empty(N, dtype=dtype), np.empty((N, D), dtype=dtype),
            np.empty((N, S), dtype=dtype, order="F"))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_single_column_matches_grad_x(ag, dtype):
    """S = 1, w = 1 on the handle's own column: every output against agp_post_logpdf_grad_x on the same handle (mbar and
    Ybar against alpha)"""
    N, D = 700, 3
    k, spec = kernel(ag, cr.MATERN52, cr.T_SCALE, D)
    X, Y = data(N, D, 1, dtype, seed=3)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), Y[:, 0])
    h = post.data.C.h
    g0, nd0, xg0 = _grad_x(ag, h, N, D, dtype)
    g, nd, md, xg, yb = _outs(N, D, 1, dtype)
    assert _cols(ag, h, np.asfortranarray(Y), g=g, nd=nd, md=md, xg=xg, yb=yb) == 0
    rt = 1e-9 if dtype == np.float64 else 1e-2
    close(g, g0, rt)
    close(nd, nd0, rt)
    close(xg, xg0, rt)
    close(md, post.data.alpha, rt)
    close(yb[:, 0], -post.data.alpha, rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_other_y_than_the_fitted_one(ag, dtype):
    """the pullback is evaluated at the Y passed, not at the handle's; mean NULL is the handle's constant mean"""
    N, D, S = 400, 2, 130
    k, spec = kernel(ag, cr.SE, cr.T_ARD, D)
    X, Y = data(N, D, S, dtype, seed=4)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), np.zeros(N, dtype=dtype))
    w = weights(S, "mixed")
    g, nd, md, xg, yb = _outs(N, D, S, dtype)
    assert _cols(ag, post.data.C.h, np.asfortranarray(Y), w=w, g=g, nd=nd, md=md, xg=xg, yb=yb) == 0
    want = lc.logpdf_grad_cols(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X.astype(np.float64), Y.astype(np.float64), w)
    rt = RT[dtype]
    close(g[0], want["grad"][0], rt)
    close(g[5:], want["grad"][5:], rt)
    close(g[3:5], want["grad"][3:5], rt)
    close(nd, want["noise_diag"], rt)
    close(md, want["mean_diag"], rt)
    close(xg, want["x"], rt)
    close(yb, want["Y"], rt)


def _additivity(ag, dtype, N, D, S, fx_of, rt):
    """w on a fit of all S columns equals sum_s w_s agp_post_logpdf_grad_x on fits of column s alone"""
    X, Y = data(N, D, S, dtype, seed=5)
    fx = fx_of(X)
    w = np.array([0.7, -1.3, 0.0, 2.1][:S])
    _, post = ag.fit(fx, Y)
    g, nd, md, xg, yb = _outs(N, D, S, dtype)
    n_cols, rc = _launches(ag, lambda: _cols(ag, post.data.C.h, np.asfortranarray(Y), w=w, g=g, nd=nd, md=md, xg=xg, yb=yb))
    assert rc == 0
    wg, wnd, wmd, wxg = np.zeros(5 + D), np.zeros(N), np.zeros(N), np.zeros((N, D))
    for s in range(S):
        ps = ag.posterior(fx, Y[:, s])
        gs, nds, xgs = _grad_x(ag, ps.data.C.h, N, D, dtype)
        wg += w[s] * gs
        wnd += w[s] * nds
        wmd += w[s] * ps.data.alpha
        wxg += w[s] * xgs
        close(yb[:, s], -w[s] * ps.data.alpha.astype(np.float64), rt)
    close(g, wg, rt)
    close(nd, wnd, rt)
    close(md, wmd, rt)
    close(xg, wxg, rt)
    return n_cols, (g, nd, md, xg, yb)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_unit_weights_add_up(ag, dtype):
    k, _ = kernel(ag, cr.MATERN12, cr.T_ARD, 3)
    _additivity(ag, dtype, 600, 3, 4, lambda X: ag.GP(0.3, k)(ag.RowVecs(X), 0.1), 1e-9 if dtype == np.float64 else 1e-2)


@pytest.mark.parametrize("dtype,N", [(np.float64, 8320), (np.float32, 4224)])
def test_int8_slice_sizes(ag, dtype, N):
    """fp64 N = 8320 and fp32 N = 4224: the factor, V = L^-1 and the column substitutions run on the int8-slice kernels.
    The branch is asserted from the launch counter (the automatic policy against tensor mode 0 on the same handle), the
    results by linearity against agp_post_logpdf_grad_x on fits of single columns"""
    eng = ag.engine()
    D, S = 2, 2
    k, _ = kernel(ag, cr.SE, cr.T_ARD, D)
    rt = 1e-8 if dtype == np.float64 else 2e-2
    n_auto, outs = _additivity(ag, dtype, N, D, S, lambda X: ag.GP(0.3, k)(ag.RowVecs(X), 0.1), rt)
    X, Y = data(N, D, S, dtype, seed=5)
    _, post = ag.fit(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), Y)
    cfg = eng.get_config()
    key = "fp64_mode" if dtype == np.float64 else "fp32_mode"
    g, nd, md, xg, yb = _outs(N, D, S, dtype)
    try:
        eng.set_config(**{key: 0})
        n_plain, rc = _launches(ag, lambda: _cols(ag, post.data.C.h, np.asfortranarray(Y), w=np.array([0.7, -1.3]), g=g, nd=nd,
                                                  md=md, xg=xg, yb=yb))
    finally:
        eng.set_config(**{key: getattr(cfg, key)})
    assert rc == 0
    assert n_auto != n_plain, (n_auto, n_plain)
    for a, b in zip((g, nd, md, xg, yb), outs):
        close(a, b, rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname,D", [("stationary", 1), ("ard", 3), ("mixed", 3)])
def test_composite(ag, dtype, kname, D):
    k = KERNELS[kname](ag, D)
    ko = oracle_of(ag, k, D)
    X, Y = data(333, D, 3, dtype, seed=6)
    X[100] = X[7]
    w = weights(3, "mixed")
    lp, g = ag.loglikelihood_grad(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), Y, lp_bar=w, inputs=True)
    want = lc.logpdf_grad_cols(ko, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X.astype(np.float64), Y.astype(np.float64), w)
    rt = RT[dtype]
    wk = ag.api._Flat(k, D).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(v, dtype=np.float64)).max() for v in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(np.asarray(a, dtype=np.float64), b, rtol=rt, atol=rt * scale)
    close(g["noise"], want["grad"][3], rt)
    close(g["mean_c"], want["grad"][4], rt)
    close(g["x"], want["x"], rt)
    close(g["Y"], want["Y"], rt)


def test_mauna_loa(ag):
    x, y = _co2()
    xtr = x[:400]
    th0 = np.array([4.0, 4.0, 0.0, 1.0, 4.0, 0.0, 0.0, -1.0, -2.0, -2.0, -2.0])
    k = _mauna_loa_kernel(ag, th0)
    ko = oracle_of(ag, k, 1)
    rng = np.random.default_rng(3)
    Y = np.stack([y[:400], y[:400] + rng.standard_normal(400), y[:400] - 1.0], axis=1)
    m = float(np.mean(y[:400]))
    lp, g = ag.loglikelihood_grad(ag.GP(m, k)(xtr, 0.05), Y, inputs=True)
    want = lc.logpdf_grad_cols(ko, ref.MeanSpec(1, m), ref.NoiseSpec(0, 0.05), xtr[:, None], Y)
    wk = ag.api._Flat(k, 1).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(v, dtype=np.float64)).max() for v in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(a, b, rtol=1e-7, atol=1e-7 * scale)
    close(g["x"], want["x"][:, 0], 1e-7)
    close(g["noise"], want["grad"][3], 1e-7)
    close(g["mean_c"], want["grad"][4], 1e-7)
    close(g["Y"], want["Y"], 1e-7)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_determinism_and_null_outputs(ag, dtype):
    """two calls give the same bits in every per-point output and in grad_out[4]; the rest of grad_out agrees to rounding;
    NULL outputs are skipped; the feature-major layout is the transpose of the point-major one"""
    N, D, S = 700, 3, 1100
    k, _ = kernel(ag, cr.MATERN32, cr.T_SCALE, D)
    X, Y = data(N, D, S, dtype, seed=7)
    _, post = ag.fit(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), Y[:, :3])
    h, Yf, w = post.data.C.h, np.asfortranarray(Y), weights(S, "mixed")
    outs = []
    for _ in range(2):
        o = _outs(N, D, S, dtype)
        assert _cols(ag, h, Yf, w=w, g=o[0], nd=o[1], md=o[2], xg=o[3], yb=o[4]) == 0
        outs.append(o)
    for a, b in zip(outs[0][1:], outs[1][1:]):
        assert a.tobytes() == b.tobytes()
    assert outs[0][0][4] == outs[1][0][4]
    np.testing.assert_allclose(outs[0][0], outs[1][0], rtol=1e-12, atol=1e-12 * np.abs(outs[0][0]).max())
    yb = np.empty((N, S), dtype=dtype, order="F")
    assert _cols(ag, h, Yf, w=w, yb=yb) == 0  # only Ybar: C^-1, the rank-S updates and the reductions are skipped
    assert yb.tobytes() == outs[0][4].tobytes()
    md = np.empty(N, dtype=dtype)
    assert _cols(ag, h, Yf, w=w, md=md) == 0
    assert md.tobytes() == outs[0][2].tobytes()
    xf = np.empty((N, D), dtype=dtype, order="F")
    assert _cols(ag, h, Yf, w=w, xg=xf, layout=1) == 0
    assert xf.tobytes(order="F") == np.asfortranarray(outs[0][3]).tobytes(order="F")
    assert _cols(ag, h, Yf, w=w) == 0  # nothing requested


def test_device_memory(ag):
    torch = pytest.importorskip("torch")
    cabi = ag._cabi
    eng = ag.engine()
    N, D, S = 500, 4, 130
    k, _ = kernel(ag, cr.SE, cr.T_ARD, D)
    X, Y = data(N, D, S, np.float64, seed=8)
    _, post = ag.fit(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), Y[:, :2])
    h, Yf, w = post.data.C.h, np.asfortranarray(Y), weights(S, "mixed")
    g0, nd0, md0, xg0, yb0 = _outs(N, D, S, np.float64)
    assert _cols(ag, h, Yf, w=w, g=g0, nd=nd0, md=md0, xg=xg0, yb=yb0) == 0
    Yd = torch.from_numpy(Yf.ravel(order="F").copy()).cuda()
    nd, md, xg, yb = (torch.empty(n, dtype=torch.float64, device="cuda") for n in (N, N, N * D, N * S))
    g = np.zeros(5 + D)
    torch.cuda.synchronize()
    eng.set_memspace(cabi.AGP_MEM_DEVICE)
    try:
        rc = _cols(ag, h, _DevArr(Yd, N, S), w=w, g=g, nd=nd.data_ptr(), md=md.data_ptr(), xg=xg.data_ptr(), yb=yb.data_ptr())
    finally:
        eng.set_memspace(cabi.AGP_MEM_HOST)
    assert rc == 0
    assert nd.cpu().numpy().tobytes() == nd0.tobytes() and md.cpu().numpy().tobytes() == md0.tobytes()
    assert xg.cpu().numpy().tobytes() == xg0.tobytes() and yb.cpu().numpy().tobytes() == yb0.tobytes(order="F")
    np.testing.assert_allclose(g, g0, rtol=1e-12, atol=1e-12 * np.abs(g0).max())


def test_errors(ag):
    cabi = ag._cabi
    N, D, S = 50, 2, 3
    k, _ = kernel(ag, cr.SE, cr.T_SCALE, D)
    X, Y = data(N, D, S, np.float64, seed=9)
    fx = ag.GP(0.3, k)(ag.RowVecs(X), 0.1)
    post = ag.posterior(fx, Y[:, 0])
    h, Yf = post.data.C.h, np.asfortranarray(Y)
    g = np.zeros(5 + D)
    assert _cols(ag, h, Yf, g=g, S=0) == cabi.AGP_ERR_INVALID
    assert _cols(ag, h, Yf, g=g, S=-2) == cabi.AGP_ERR_INVALID
    assert _cols(ag, h, None, g=g) == cabi.AGP_ERR_INVALID
    assert _cols(ag, h, Yf, g=g, layout=2) == cabi.AGP_ERR_INVALID
    assert _cols(ag, h, Yf, g=g, mean=cabi.agp_mean(2, 0.0, None)) == cabi.AGP_ERR_INVALID
    assert ag.engine().L.agp_post_logpdf_grad_cols(None, None, cabi.ptr(Yf), S, None, None, None, None, 0, None, None) == \
        cabi.AGP_ERR_INVALID
    # a handle extended by sequential conditioning
    X2, Y2 = data(20, D, 1, np.float64, seed=10)
    post2 = ag.posterior(post(ag.RowVecs(X2), 0.1), Y2[:, 0])
    Y12 = np.asfortranarray(np.vstack([Y, np.repeat(Y2, S, axis=1)]))
    assert _cols(ag, post2.data.C.h, Y12, g=np.zeros(5 + D)) == cabi.AGP_ERR_UNSUPPORTED
    # the handle still works, and a vector mean passed again matches the constant it equals
    g1, g2 = np.zeros(5 + D), np.zeros(5 + D)
    assert _cols(ag, h, Yf, g=g1) == 0
    mv = np.full(N, 0.3)
    assert _cols(ag, h, Yf, g=g2, mean=cabi.agp_mean(2, 0.0, mv.ctypes.data)) == 0
    np.testing.assert_allclose(g1, g2, rtol=1e-12, atol=1e-12 * np.abs(g1).max())


# ---- the reference's matrix cases (test/finite_gp_projection.jl:128-178) -----------------------------------------------
def test_reference_matrix_logpdf_gradients(ag):
    """f = GP(1, SE), N = 10, S = 11: the x-gradient of l * sum(logpdf(f(x, 1e-3), ones(N, S))) and the (sigma_, Y)-gradient
    of l * sum(logpdf(f(x, exp(sigma_)), Y)), against torch fp64 autograd and central differences of agp_fit"""
    torch = pytest.importorskip("torch")
    N, S = 10, 11
    rng = np.random.default_rng(123456)
    x, lbar, sig = rng.standard_normal(N), rng.standard_normal(), rng.standard_normal()
    Yh = rng.standard_normal((N, S))
    f = ag.GP(1.0, ag.SqExponentialKernel())

    def torch_lp(xt, s2, Yt):
        C_ = torch.exp(-0.5 * (xt[:, None] - xt[None, :]) ** 2) + s2 * torch.eye(N, dtype=torch.float64)
        L = torch.linalg.cholesky(C_)
        Zq = torch.linalg.solve_triangular(L, Yt - 1.0, upper=False)
        return -0.5 * (N * np.log(2 * np.pi) + 2 * torch.log(torch.diagonal(L)).sum() + (Zq * Zq).sum(0))

    # x -> sum(logpdf(f(x, 1e-3), ones(N, S)))
    ones = np.ones((N, S))
    _, g = ag.loglikelihood_grad(f(x, 1e-3), ones, lp_bar=np.full(S, lbar), inputs=True)
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    (lbar * torch_lp(xt, 1e-3, torch.as_tensor(ones)).sum()).backward()
    np.testing.assert_allclose(g["x"], xt.grad.numpy(), rtol=1e-8, atol=1e-8)
    h = 1e-6
    for i in (0, 4, 9):
        xp, xm = x.copy(), x.copy()
        xp[i] += h
        xm[i] -= h
        fd = lbar * (ag.loglikelihood(f(xp, 1e-3), ones) - ag.loglikelihood(f(xm, 1e-3), ones)) / (2 * h)
        assert abs(g["x"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, g["x"][i], fd)
    # (sigma_, Y) -> sum(logpdf(f(x, exp(sigma_)), Y))
    _, g = ag.loglikelihood_grad(f(x, np.exp(sig)), Yh, lp_bar=np.full(S, lbar))
    st = torch.tensor(sig, dtype=torch.float64, requires_grad=True)
    Yt = torch.tensor(Yh, dtype=torch.float64, requires_grad=True)
    (lbar * torch_lp(torch.as_tensor(x), torch.exp(st), Yt).sum()).backward()
    np.testing.assert_allclose(g["noise"] * np.exp(sig), st.grad.item(), rtol=1e-8, atol=1e-8)
    np.testing.assert_allclose(g["Y"], Yt.grad.numpy(), rtol=1e-8, atol=1e-8)
    fd = lbar * (ag.loglikelihood(f(x, np.exp(sig + h)), Yh) - ag.loglikelihood(f(x, np.exp(sig - h)), Yh)) / (2 * h)
    assert abs(g["noise"] * np.exp(sig) - fd) <= 1e-6 * max(1.0, abs(fd))
    Yp, Ym = Yh.copy(), Yh.copy()
    Yp[3, 5] += h
    Ym[3, 5] -= h
    fd = lbar * (ag.loglikelihood(f(x, np.exp(sig)), Yp) - ag.loglikelihood(f(x, np.exp(sig)), Ym)) / (2 * h)
    assert abs(g["Y"][3, 5] - fd) <= 1e-6 * max(1.0, abs(fd))
