"""The pullback of rand over an exact posterior on the device (agp_post_rand_grad), in fp64 and fp32: against the CPU
model tests/post_rand_grad_ref.py for the five single-kernel families under every transform in the row, column and vector
containers, per-point noises and vector means, composites and the Mauna Loa kernel on a train / test split of the CO2
data; the samples against the model and agp_post_rand; central differences of agp_post_rand over refits; the multi-column
backward substitution on its tile and int8-slice schedules, the branch asserted from the launch counter; device memory,
determinism, NULL outputs, the error codes; and an L-BFGS-B replay of a fixed-normals Monte Carlo expected improvement
maximised over the candidate points.
Tolerances: rtol 1e-7 (fp64) / 2e-2 (fp32, against the model on the fp32-rounded inputs), atol the same times max|g|."""
import ctypes as C

import numpy as np
import pytest

import composite_ref as cr
import post_rand_grad_ref as prr
from oracle import agp_ref as ref
from test_gpu_composite import KERNELS, _co2, _mauna_loa_kernel, oracle_of
from test_gpu_rand_grad import _DevArr, _launches, check_single, close, container, kernel, x_rows

pytestmark = pytest.mark.gpu
RT = {np.float64: 1e-7, np.float32: 2e-2}
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]
TILE = 128


def data(N, M, D, S, dtype, seed=0):
    rng = np.random.default_rng(seed + 7 * N + 3 * M + D + 5 * S)
    return (rng.uniform(-2, 2, (N, D)).astype(dtype), rng.standard_normal(N).astype(dtype),
            rng.uniform(-2.2, 2.2, (M, D)).astype(dtype), rng.standard_normal((M, S)).astype(dtype),
            rng.standard_normal((M, S)).astype(dtype))


def f64(*a):
    return [np.asarray(v, dtype=np.float64) for v in a]


def close_sum(got, want, terms, rt):
    """a scalar that is a sum of terms, to rt of the sum of their magnitudes: the training noise entry is tr(Cbar) and
    the ConstMean entry sum mubar - sum beta, and at N = 1300, M = 1000 their terms cancel to 1 part in ~100 (an fp32
    evaluation of the model's formulas on the CPU is 12% off the fp64 one there)"""
    scale = float(np.sum(np.abs(np.asarray(terms, dtype=np.float64))))
    np.testing.assert_allclose(float(got), float(want), rtol=rt, atol=rt * scale)


def check_all(out, g, want, spec, kind, rt, kernel=True):
    close(out, want["out"], rt)
    if kernel:
        check_single(g, want, spec, rt)
    close_sum(g["noise"], want["grad"][3], want["noise_diag"], rt)
    close_sum(g["mean_c"], want["grad"][4], np.concatenate([want["mean_s_diag"], want["y"]]), rt)
    close(g["noise_s"], np.sum(want["noise_s_diag"]), rt)
    close(g["y"], want["y"], rt)
    close(g["Z"], want["Z"], rt)
    close(x_rows(g["x"], kind), want["x"], rt)
    close(x_rows(g["xs"], kind), want["xs"], rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_matches_model(ag, family, transform, dtype):
    rt = RT[dtype]
    for N, M, D, S, kind in [(1, 1, 1, 1, "vec"), (63, 17, 3, 2, "row"), (333, 129, 1, 3, "col"), (333, 200, 40, 2, "row"),
                             (1300, 1000, 3, 64, "col")]:
        k, spec = kernel(ag, family, transform, D)
        X, y, Xs, Z, Ob = data(N, M, D, S, dtype)
        p = ag.posterior(ag.GP(0.3, k)(container(ag, X, kind), 0.1), y)
        fx = p(container(ag, Xs, kind), 0.05)
        out, g = ag.posterior_rand_grad(fx, Z, Ob, inputs=True)
        want = prr.post_rand_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs),
                                  ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.05), *f64(Z, Ob))
        assert g["xs"].dtype == dtype and g["Z"].dtype == dtype and g["Z"].shape == (M, S)
        # fp32 Linear kernel gradients are differences of nearly equal terms (the posterior covariance of a rank-D prior is
        # the test noise plus O(D / N)), as for the held-out gradient (DESIGN s6): held to the model in fp64 only
        linear32 = spec.family == cr.LINEAR and dtype == np.float32
        check_all(out, g, want, spec, kind, rt, kernel=not linear32)
        assert out.tobytes() == ag.api._post_rand_from_normals(fx, Z).tobytes()  # the samples are agp_post_rand's


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_per_point_noises_and_vector_means(ag, dtype):
    N, M, D, S = 500, 300, 2, 5
    k, spec = kernel(ag, cr.MATERN32, cr.T_ARD, D)
    X, y, Xs, Z, Ob = data(N, M, D, S, dtype, seed=2)
    rng = np.random.default_rng(2)
    s2, s2s = rng.uniform(0.05, 0.2, N), rng.uniform(0.02, 0.1, M)
    p = ag.posterior(ag.GP(ag.CustomMean(lambda x: np.sin(x[0])), k)(ag.RowVecs(X), s2), y)
    out, g = ag.posterior_rand_grad(p(ag.RowVecs(Xs), s2s), Z, Ob, inputs=True)
    r = lambda a: np.asarray(a).astype(dtype).astype(np.float64)  # noqa: E731
    X64, Xs64 = f64(X, Xs)
    want = prr.post_rand_grad(spec, ref.MeanSpec(2, v=r(np.sin(X64[:, 0]))), ref.NoiseSpec(1, v=r(s2)), X64, *f64(y), Xs64,
                              ref.MeanSpec(2, v=r(np.sin(Xs64[:, 0]))), ref.NoiseSpec(1, v=r(s2s)), *f64(Z, Ob))
    rt = RT[dtype]
    close(out, want["out"], rt)
    for key, wk in [("noise", "noise_diag"), ("mean_v", "mean_diag"), ("noise_s", "noise_s_diag"),
                    ("mean_s_v", "mean_s_diag"), ("x", "x"), ("xs", "xs"), ("y", "y"), ("Z", "Z")]:
        close(g[key], want[wk], rt)
    check_single(g, want, spec, rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname,D", [("stationary", 1), ("ard", 3), ("mixed", 3)])
def test_composite(ag, dtype, kname, D):
    k = KERNELS[kname](ag, D)
    ko = oracle_of(ag, k, D)
    X, y, Xs, Z, Ob = data(333, 150, D, 3, dtype, seed=6)
    p = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    out, g = ag.posterior_rand_grad(p(ag.RowVecs(Xs), 0.05), Z, Ob, inputs=True)
    want = prr.post_rand_grad(ko, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs), ref.MeanSpec(1, 0.3),
                              ref.NoiseSpec(0, 0.05), *f64(Z, Ob))
    rt = RT[dtype]
    wk = ag.api._Flat(k, D).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(v, dtype=np.float64)).max() for v in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(np.asarray(a, dtype=np.float64), b, rtol=rt, atol=rt * scale)
    for key in ("x", "xs", "y", "Z"):
        close(g[key], want[key], rt)
    close(g["noise"], want["grad"][3], rt)
    close(g["mean_c"], want["grad"][4], rt)
    close(out, want["out"], rt)


def test_mauna_loa_forecast(ag):
    """the Mauna Loa kernel on the CO2 data: train on the first 400 months, sample the next 150"""
    x, y = _co2()
    xtr, ytr, xte = x[:400], y[:400], x[400:550]
    k = _mauna_loa_kernel(ag, np.array([4.0, 4.0, 0.0, 1.0, 4.0, 0.0, 0.0, -1.0, -2.0, -2.0, -2.0]))
    ko = oracle_of(ag, k, 1)
    m = float(np.mean(ytr))
    rng = np.random.default_rng(21)
    Z, Ob = rng.standard_normal((150, 8)), rng.standard_normal((150, 8))
    p = ag.posterior(ag.GP(m, k)(xtr, 0.05), ytr)
    out, g = ag.posterior_rand_grad(p(xte, 0.05), Z, Ob, inputs=True)
    want = prr.post_rand_grad(ko, ref.MeanSpec(1, m), ref.NoiseSpec(0, 0.05), xtr[:, None], ytr, xte[:, None], ref.MeanSpec(1, m),
                              ref.NoiseSpec(0, 0.05), Z, Ob)
    wk = ag.api._Flat(k, 1).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(v, dtype=np.float64)).max() for v in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(a, b, rtol=1e-7, atol=1e-7 * scale)
    close(out, want["out"], 1e-9)
    close(g["x"], want["x"][:, 0], 1e-7)
    close(g["xs"], want["xs"][:, 0], 1e-7)
    close(g["noise"], want["grad"][3], 1e-7)
    close(g["noise_s"], np.sum(want["noise_s_diag"]), 1e-7)
    close(g["mean_c"], want["grad"][4], 1e-7)
    close(g["y"], want["y"], 1e-7)
    close(g["Z"], want["Z"], 1e-7)


def test_central_differences_over_refits(ag):
    """the kernel scale, the training noise, an input, a target, a test input and a normal against central differences of
    agp_post_rand over refits"""
    N, M, D, S = 120, 40, 2, 3
    X, y, Xs, Z, Ob = data(N, M, D, S, np.float64, seed=11)
    ls, s2 = 0.9, 0.1

    def F(ls_=ls, s2_=s2, X_=X, y_=y, Xs_=Xs, Z_=Z):
        k = ag.with_lengthscale(ag.Matern52Kernel(), ls_)
        p = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X_), s2_), y_)
        return float(np.sum(Ob * ag.api._post_rand_from_normals(p(ag.RowVecs(Xs_), 0.05), Z_)))
    p = ag.posterior(ag.GP(0.3, ag.with_lengthscale(ag.Matern52Kernel(), ls))(ag.RowVecs(X), s2), y)
    out, g = ag.posterior_rand_grad(p(ag.RowVecs(Xs), 0.05), Z, Ob, inputs=True)
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
    Zp, Zm = Z.copy(), Z.copy()
    Zp[5, 2] += h
    Zm[5, 2] -= h
    v = fd(F(Z_=Zp), F(Z_=Zm))
    assert abs(g["Z"][5, 2] - v) <= 1e-6 * max(1.0, abs(v)), (g["Z"][5, 2], v)


# ---- the raw entry point on a handle -----------------------------------------------------------------------------------
def _call(ag, h, Xs, Z, Ob, S=None, outs=None, layout=0, mean=None, noise=None, M=None):
    eng = ag.engine()
    p = lambda a: a if isinstance(a, int) else ag._cabi.ptr(a)  # noqa: E731
    dp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    o = outs or {}
    M = (Xs.shape[0] if layout == 0 else Xs.shape[-1]) if M is None else M
    S = (Z.shape[1] if Z is not None else 1) if S is None else S
    return eng.L.agp_post_rand_grad(
        h, layout, p(Xs), M, None if mean is None else C.byref(mean), None if noise is None else C.byref(noise), p(Z), S,
        p(Ob), dp(o.get("g")), p(o.get("nd")), p(o.get("md")), p(o.get("yb")), p(o.get("xg")), p(o.get("nsd")),
        p(o.get("msd")), p(o.get("zb")), p(o.get("xsg")))


def _outs(N, M, D, S, dtype, glen=None):
    e = lambda *s: np.empty(s, dtype=dtype, order="F")  # noqa: E731
    # the input gradients point-major: D x n column-major, i.e. n x D row-major
    return dict(g=np.zeros(5 + D if glen is None else glen), nd=e(N), md=e(N), yb=e(N), xg=np.empty((N, D), dtype=dtype),
                nsd=e(M), msd=e(M), zb=e(M, S), xsg=np.empty((M, D), dtype=dtype))


def _noise(ag, s):
    return ag._cabi.agp_noise(0, s, None)


def _subst_case(ag, dtype, N, M, key, mode):
    """the fit and the calls under `key` = mode, then again under 0 (the tile kernels).  The launches of the training side
    are the difference between a call that asks for y_bar only (P = L^-T A, then beta) and one that asks for z_bar only
    (the same forward and head, no P): on the tile schedule that is 2 nblk - 1 GEMMs for the substitution plus a fixed
    number for beta, and the int8-slice schedule differs from it.  Both agree with the model."""
    eng = ag.engine()
    D, S = 2, 3
    k, spec = kernel(ag, cr.SE, cr.T_ARD, D)
    X, y, Xs, Z, Ob = data(N, M, D, S, dtype, seed=12)
    Zf, Of, Xsc = np.asfortranarray(Z), np.asfortranarray(Ob), np.ascontiguousarray(Xs)
    nblk = -(-N // TILE)
    cfg = eng.get_config()
    res = []
    try:
        for m in (mode, 0):
            eng.set_config(**{key: m})  # before the fit: the handle's own factor comes from this policy too
            post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
            h = post.data.C.h
            n_z, rc = _launches(ag, lambda: _call(ag, h, Xsc, Zf, Of, outs=dict(zb=np.empty((M, S), dtype=dtype, order="F")),
                                                  noise=_noise(ag, 0.05)))
            assert rc == 0
            n_y, rc = _launches(ag, lambda: _call(ag, h, Xsc, Zf, Of, outs=dict(yb=np.empty(N, dtype=dtype)),
                                                  noise=_noise(ag, 0.05)))
            assert rc == 0
            o = _outs(N, M, D, S, dtype)
            assert _call(ag, h, Xsc, Zf, Of, outs=o, noise=_noise(ag, 0.05)) == 0
            res.append((n_y - n_z, o))
    finally:
        eng.set_config(**{key: getattr(cfg, key)})
    tc, tile = res[0][0], res[1][0]
    beta = tile - (2 * nblk - 1)
    assert 0 < beta <= 4, (tile, nblk)
    assert tc != tile, (tc, tile)
    want = prr.post_rand_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), *f64(X, y, Xs), ref.MeanSpec(1, 0.3),
                              ref.NoiseSpec(0, 0.05), *f64(Z, Ob))
    rt = RT[dtype]
    for _, o in res:
        for key_, wk in [("nd", "noise_diag"), ("yb", "y"), ("xg", "x"), ("nsd", "noise_s_diag"), ("msd", "mean_s_diag"),
                         ("zb", "Z"), ("xsg", "xs")]:
            close(o[key_], want[wk], rt)
        close(o["g"][[0, 5, 6]], want["grad"][[0, 5, 6]], rt)
        close_sum(o["g"][3], want["grad"][3], want["noise_diag"], rt)
        close_sum(o["g"][4], want["grad"][4], np.concatenate([want["mean_s_diag"], want["y"]]), rt)


def test_backward_substitution_forced_fp64(ag):
    """fp64 at N = 2304, M = 512 with the int8-slice kernels forced (fp64_mode = 1): the rank-512 updates of the backward
    substitution run on the int8-slice kernel, the ragged outer block on the tile GEMM"""
    _subst_case(ag, np.float64, 2304, 512, "fp64_mode", 1)


@pytest.mark.parametrize("dtype,N,key", [(np.float64, 8320, "fp64_mode"), (np.float32, 4224, "fp32_mode")])
def test_backward_substitution_automatic(ag, dtype, N, key):
    """fp64 N = 8320 and fp32 N = 4224, M = 600: the automatic policy (-1) takes the int8-slice kernels"""
    _subst_case(ag, dtype, N, 600, key, -1)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_determinism_null_outputs_and_layouts(ag, dtype):
    N, M, D, S = 700, 300, 3, 130
    k, _ = kernel(ag, cr.MATERN32, cr.T_SCALE, D)
    X, y, Xs, Z, Ob = data(N, M, D, S, dtype, seed=7)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Zf, Of, Xsc = post.data.C.h, np.asfortranarray(Z), np.asfortranarray(Ob), np.ascontiguousarray(Xs)
    outs = []
    for _ in range(2):
        o = _outs(N, M, D, S, dtype)
        assert _call(ag, h, Xsc, Zf, Of, outs=o, noise=_noise(ag, 0.05)) == 0
        outs.append(o)
    for key in outs[0]:
        if key != "g":
            assert outs[0][key].tobytes() == outs[1][key].tobytes(), key
    assert outs[0]["g"][3:5].tobytes() == outs[1]["g"][3:5].tobytes()
    np.testing.assert_allclose(outs[0]["g"], outs[1]["g"], rtol=1e-10, atol=1e-10 * np.abs(outs[0]["g"]).max())
    for key in ("zb", "msd", "yb", "md", "xsg", "nsd"):  # each alone: the rest of the work is skipped, the bits are the same
        o = {key: np.empty_like(outs[0][key])}
        assert _call(ag, h, Xsc, Zf, Of, outs=o, noise=_noise(ag, 0.05)) == 0
        assert o[key].tobytes() == outs[0][key].tobytes(), key
    # feature-major: the input points and both input gradients as M x D / N x D column-major
    o = dict(xg=np.empty((N, D), dtype=dtype, order="F"), xsg=np.empty((M, D), dtype=dtype, order="F"))
    assert _call(ag, h, np.asfortranarray(Xs), Zf, Of, outs=o, layout=1, M=M, noise=_noise(ag, 0.05)) == 0
    assert o["xg"].tobytes(order="F") == np.asfortranarray(outs[0]["xg"]).tobytes(order="F")
    assert o["xsg"].tobytes(order="F") == np.asfortranarray(outs[0]["xsg"]).tobytes(order="F")
    assert _call(ag, h, Xsc, Zf, Of) == 0  # nothing requested


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_device_memory(ag, dtype):
    torch = pytest.importorskip("torch")
    cabi = ag._cabi
    eng = ag.engine()
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    N, M, D, S = 500, 200, 4, 33
    k, _ = kernel(ag, cr.SE, cr.T_ARD, D)
    X, y, Xs, Z, Ob = data(N, M, D, S, dtype, seed=8)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Zf, Of, Xsc = post.data.C.h, np.asfortranarray(Z), np.asfortranarray(Ob), np.ascontiguousarray(Xs)
    o0 = _outs(N, M, D, S, dtype)
    assert _call(ag, h, Xsc, Zf, Of, outs=o0, noise=_noise(ag, 0.05)) == 0
    Zd = torch.from_numpy(Zf.ravel(order="F").copy()).cuda()
    Od = torch.from_numpy(Of.ravel(order="F").copy()).cuda()
    Xd = torch.from_numpy(Xsc.ravel().copy()).cuda()
    dev = {key: torch.empty(v.size, dtype=tdt, device="cuda") for key, v in o0.items() if key != "g"}
    o = {key: t.data_ptr() for key, t in dev.items()}
    o["g"] = np.zeros(5 + D)
    torch.cuda.synchronize()
    eng.set_memspace(cabi.AGP_MEM_DEVICE)
    try:
        rc = _call(ag, h, _DevArr(Xd, M, D), _DevArr(Zd, M, S), _DevArr(Od, M, S), outs=o, M=M, noise=_noise(ag, 0.05))
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
    X, y, Xs, Z, Ob = data(N, M, D, S, np.float64, seed=9)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h, Zf, Of, Xsc = post.data.C.h, np.asfortranarray(Z), np.asfortranarray(Ob), np.ascontiguousarray(Xs)
    g = dict(g=np.zeros(5 + D))
    assert _call(ag, h, Xsc, Zf, Of, outs=g, S=0) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Zf, Of, outs=g, S=-2) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, None, Of, outs=g, S=S) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Zf, None, outs=g) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, None, Zf, Of, outs=g, M=M) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Zf, Of, outs=g, layout=2) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Zf, Of, outs=g, mean=cabi.agp_mean(2, 0.0, None)) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Zf, Of, outs=g, noise=cabi.agp_noise(1, 0.0, None)) == cabi.AGP_ERR_INVALID
    assert _call(ag, h, Xsc, Zf, Of, outs=g, M=0) == cabi.AGP_ERR_DIM_MISMATCH
    # a test covariance that is not positive definite: a negative test noise larger than the posterior variance
    assert _call(ag, h, Xsc, Zf, Of, outs=g, noise=_noise(ag, -5.0)) == cabi.AGP_ERR_NOT_POSDEF
    assert ag.engine().L.agp_last_info(ag.engine().h) > 0
    assert ag.engine().L.agp_post_rand_grad(None, 0, cabi.ptr(Xsc), M, None, None, cabi.ptr(Zf), S, cabi.ptr(Of),
                                            *([None] * 9)) == cabi.AGP_ERR_INVALID
    X2, y2, _, _, _ = data(20, 1, D, 1, np.float64, seed=10)
    post2 = ag.posterior(post(ag.RowVecs(X2), 0.1), y2)
    assert _call(ag, post2.data.C.h, Xsc, Zf, Of, outs=dict(g=np.zeros(5 + D))) == cabi.AGP_ERR_UNSUPPORTED
    o = _outs(N, M, D, S, np.float64)  # the handle still works after every refusal
    assert _call(ag, h, Xsc, Zf, Of, outs=o) == 0
    assert np.all(np.isfinite(o["g"]))


def test_lbfgs_monte_carlo_expected_improvement_replay(ag):
    """a smoothed q-EI with fixed normals: L-BFGS-B over a batch of q = 3 candidate points x*, maximising
    mean_s (1/tau) log(1 + sum_m exp(tau (out[m, s] - best))), out = rand over the posterior at the candidates, with the
    device gradient and with the model's: the two paths agree"""
    from scipy.optimize import minimize
    N, q, S, tau = 60, 3, 64, 10.0
    rng = np.random.default_rng(17)
    X = rng.uniform(-2, 2, (N, 1))
    y = np.sin(2 * X[:, 0]) + 0.1 * rng.standard_normal(N)
    best = float(np.max(y))
    Z = rng.standard_normal((q, S))
    k = 1.2 * ag.with_lengthscale(ag.SqExponentialKernel(), 0.6)
    spec = ref.KernelSpec(cr.SE, 1.2, cr.T_SCALE, 1.0 / 0.6)
    p = ag.posterior(ag.GP(k)(X[:, 0], 0.01), y)

    def ei_and_bar(out):
        e = np.exp(tau * (out - best))
        v = np.log1p(e.sum(axis=0)) / tau
        return float(np.mean(v)), e / (1.0 + e.sum(axis=0)) / S

    def dev(xs):
        fx = p(xs, 1e-6)
        v, Ob = ei_and_bar(ag.api._post_rand_from_normals(fx, Z))
        _, g = ag.posterior_rand_grad(fx, Z, Ob, inputs=True)
        return -v, -np.asarray(g["xs"], dtype=np.float64)

    def model(xs):
        args = (spec, ref.MeanSpec(), ref.NoiseSpec(0, 0.01), X, y, xs[:, None], ref.MeanSpec(), ref.NoiseSpec(0, 1e-6), Z)
        v, Ob = ei_and_bar(prr.post_rand_grad(*args, np.zeros((q, S)))["out"])
        return -v, -prr.post_rand_grad(*args, Ob)["xs"][:, 0]
    x0 = np.array([-1.5, 0.2, 1.4])
    paths = []
    for fun in (dev, model):
        path = []
        res = minimize(fun, x0, jac=True, method="L-BFGS-B", bounds=[(-2, 2)] * q, callback=lambda t: path.append(t.copy()),
                       options=dict(maxiter=8))
        paths.append((np.array(path), res.fun))
    assert len(paths[0][0]) == len(paths[1][0]) > 2
    np.testing.assert_allclose(paths[0][0], paths[1][0], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(paths[0][1], paths[1][1], rtol=1e-8)
