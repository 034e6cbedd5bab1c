"""The pullback of mean_and_var over an exact posterior (agp_post_mean_var_grad) without a GPU: the NumPy model
tests/post_mean_var_grad_ref.py pinned to torch fp64 autograd through torch.linalg.cholesky, with every hyper-parameter,
both noises, both means, both input sets and y as leaves; y and x* by central differences; a test point on a training
point; the Python mirror's argument passing through a stand-in library; and the structure and ccall arity of the Julia
rule."""
import ctypes as C

import numpy as np
import pytest

import composite_ref as cr
import fake_libagp
import grad_x_ref as gx
import post_mean_var_grad_ref as pmv
from oracle import agp_ref as ref
from test_api_composite_fake import CompositeFakeLib
from test_grad_x_model import mauna_loa_shape
from test_pred_logpdf_grad_model import (PRIMAL_FIELDS, _header_arity, _julia, _rule, _tangent_fields, close, problem,
                                         specs)
from test_rand_grad_model import _leaf, _torch_factor, single

FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]


def torch_pullback(k, mean, mean_s, noise, noise_s, X, y, Xs, mbar, vbar):
    """autograd of sum(mbar o mu*) + sum(vbar o sigma^2) over posterior(fx, y)(x*, Sigma*): (means, variances,
    descriptor-order kernel gradient, training noise, mean, x, y, test noise, mean, x*); a constant mean is one leaf
    shared by both sides"""
    torch = pytest.importorskip("torch")
    kc = gx.as_composite(k)
    N, M = X.shape[0], Xs.shape[0]
    Xt, Xst, yt = _leaf(torch, X), _leaf(torch, Xs), _leaf(torch, y)
    Xc = torch.cat([Xt, Xst])
    leaves = []
    K = torch.zeros((N + M, N + M), dtype=torch.float64)
    for v, fs in zip(kc.variance, kc.factors):
        vt = _leaf(torch, v)
        leaves.append(vt)
        P = vt * torch.ones((N + M, N + M), dtype=torch.float64)
        for F in fs:
            P = P * _torch_factor(torch, F, Xc, leaves)
        K = K + P
    Kxx, Kxs, Kss = K[:N, :N], K[:N, N:], K[N:, N:]
    s2 = _leaf(torch, noise.s if noise.kind == 0 else noise.v)
    s2s = _leaf(torch, noise_s.s if noise_s.kind == 0 else noise_s.v)
    if mean.kind == 1:
        mt = mst = _leaf(torch, mean.c)
    else:
        mt = _leaf(torch, mean.v if mean.kind == 2 else 0.0)
        mst = _leaf(torch, mean_s.v if mean_s.kind == 2 else 0.0)
    m = mt * torch.ones(N, dtype=torch.float64)
    ms = mst * torch.ones(M, dtype=torch.float64)
    L = torch.linalg.cholesky(Kxx + torch.diag(s2 * torch.ones(N, dtype=torch.float64)))
    alpha = torch.cholesky_solve((yt - m)[:, None], L)[:, 0]
    mu = ms + Kxs.T @ alpha
    A = torch.linalg.solve_triangular(L, Kxs, upper=False)
    var = torch.diagonal(Kss) - (A * A).sum(0) + s2s * torch.ones(M, dtype=torch.float64)
    (mu * torch.as_tensor(mbar) + var * torch.as_tensor(vbar)).sum().backward()
    kg = np.concatenate([np.atleast_1d(t.grad.numpy()) for t in leaves])
    g = lambda t: None if t.grad is None else t.grad.numpy()  # noqa: E731
    return (mu.detach().numpy(), var.detach().numpy(), kg, g(s2), g(mt), Xt.grad.numpy(), yt.grad.numpy(), g(s2s), g(mst),
            Xst.grad.numpy())


def cotangents(M, seed):
    rng = np.random.default_rng(seed + 31 * M)
    return rng.standard_normal(M), rng.standard_normal(M)


def _check(k, mean, mean_s, noise, noise_s, X, y, Xs, mbar, vbar):
    got = pmv.post_mean_var_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, mbar, vbar)
    mu, var, kg, ng, mg, xg, yg, nsg, msg, xsg = torch_pullback(k, mean, mean_s, noise, noise_s, X, y, Xs, mbar, vbar)
    close(got["mean"], mu)
    close(got["var"], var)
    if isinstance(k, cr.Composite):
        close(got["grad"][5:], kg)
    else:  # descriptor order of one factor: variance, Scale s | ARD v, Linear c
        g = got["grad"]
        want = [g[0]] + ([g[1]] if k.transform == cr.T_SCALE else []) + (list(g[5:]) if k.transform == cr.T_ARD else [])
        want += [g[2]] if k.family == cr.LINEAR else []
        close(np.array(want), kg)
    close(got["noise_diag"] if noise.kind == 1 else got["grad"][3], ng)
    close(got["noise_s_diag"] if noise_s.kind == 1 else np.sum(got["noise_s_diag"]), nsg)
    if mean.kind == 1:
        close(got["grad"][4], mg)
    elif mean.kind == 2:
        close(got["mean_diag"], mg)
        close(got["mean_s_diag"], msg)
    close(got["x"], xg)
    close(got["xs"], xsg)
    close(got["y"], yg)


@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_model_matches_torch_autograd(family, transform):
    D = 3
    k = single(family, transform, D, np.random.default_rng(family + 3 * transform))
    for M in (1, 7, 130):
        for noise_kind in (0, 1):
            for mean_kind in (0, 1, 2):
                N = 24 + 2 * mean_kind + noise_kind
                X, y, Xs, _ = problem(N, M, D, 1, seed=family + mean_kind)
                if family == cr.LINEAR:  # a rank-D kernel: shorter inputs keep C's conditioning near the others'
                    X, Xs = 0.5 * X, 0.5 * Xs
                mean, mean_s, noise, noise_s = specs(mean_kind, noise_kind, N, M, mean_kind + 3 * noise_kind)
                mbar, vbar = cotangents(M, family + noise_kind + mean_kind)
                _check(k, mean, mean_s, noise, noise_s, X, y, Xs, mbar, vbar)
    # one cotangent zero: the other output alone
    X, y, Xs, _ = problem(20, 9, D, 1, seed=family)
    mean, mean_s, noise, noise_s = specs(1, 0, 20, 9, 2)
    mbar, vbar = cotangents(9, family)
    _check(k, mean, mean_s, noise, noise_s, X, y, Xs, np.zeros(9), vbar)
    _check(k, mean, mean_s, noise, noise_s, X, y, Xs, mbar, np.zeros(9))


@pytest.mark.parametrize("D", [1, 3])
def test_model_matches_torch_autograd_mauna_loa(D):
    X, y, Xs, _ = problem(30, 12, D, 1, seed=6)
    mean, mean_s, noise, noise_s = specs(2, 1, 30, 12, D)
    mbar, vbar = cotangents(12, D)
    _check(mauna_loa_shape(D, np.random.default_rng(D)), mean, mean_s, noise, noise_s, X, y, Xs, mbar, vbar)


def linear_product(D, rng):
    """Linear x SE (Scale) + an ARD Linear alone + Matern 3/2: the kdiag term through the product rule and on its own"""
    F = cr.Factor
    return cr.Composite([0.7, 0.4, 0.9],
                        [[F(cr.LINEAR, param=0.3), F(cr.SE, cr.T_SCALE, 0.6)],
                         [F(cr.LINEAR, cr.T_ARD, ard=rng.uniform(0.5, 1.2, D), param=0.2)],
                         [F(cr.MATERN32, cr.T_SCALE, 0.8)]])


@pytest.mark.parametrize("M", [1, 7])
def test_model_matches_torch_autograd_linear_in_a_product(M):
    D = 2
    X, y, Xs, _ = problem(26, M, D, 1, seed=3)
    mean, mean_s, noise, noise_s = specs(1, 1, 26, M, 4)
    mbar, vbar = cotangents(M, 5)
    k = linear_product(D, np.random.default_rng(7))
    _check(k, mean, mean_s, noise, noise_s, 0.5 * X, y, 0.5 * Xs, mbar, vbar)
    # the kernel has a nonzero d1k(x*_j, x*_j): the kdiag term is exercised
    kd = gx.kernel_d1(k, 0.5 * Xs, 0.5 * Xs)[np.arange(M), np.arange(M)]
    assert np.abs(kd).max() > 0.1


def test_y_and_xs_match_central_differences():
    """ybar and the x* gradient against central differences of the oracle's posterior mean_and_var over refits"""
    k = single(cr.MATERN52, cr.T_ARD, 2, np.random.default_rng(0))
    X, y, Xs, _ = problem(25, 9, 2, 1, seed=9)
    mean, mean_s, noise, noise_s = specs(1, 0, 25, 9, 1)
    mbar, vbar = cotangents(9, 2)
    got = pmv.post_mean_var_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, mbar, vbar)

    def f(yy, XX):
        m, v = ref.post_mean_and_var(ref.posterior(k, mean, noise, X, yy), XX, mean_s=mean_s, noise_s=noise_s)
        return float(np.dot(mbar, m) + np.dot(vbar, v))
    h = 1e-6
    for i in (0, 7, 24):
        yp, ym = y.copy(), y.copy()
        yp[i] += h
        ym[i] -= h
        fd = (f(yp, Xs) - f(ym, Xs)) / (2 * h)
        assert abs(got["y"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, got["y"][i], fd)
    for i, d in [(0, 0), (4, 1), (8, 0)]:
        Xp, Xm = Xs.copy(), Xs.copy()
        Xp[i, d] += h
        Xm[i, d] -= h
        fd = (f(y, Xp) - f(y, Xm)) / (2 * h)
        assert abs(got["xs"][i, d] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, d, got["xs"][i, d], fd)


@pytest.mark.parametrize("family", FAMILIES)
def test_test_point_on_a_training_point_is_finite(family):
    """x*_0 = x_3: every stationary factor's pair adds exactly 0 (Matern 1/2: its zero subgradient), nothing is NaN; for the
    smooth families the result is the derivative (central differences)"""
    k = single(family, cr.T_SCALE, 2, np.random.default_rng(1))
    X, y, Xs, _ = problem(20, 4, 2, 1, seed=5)
    Xs[0] = X[3]
    mean, mean_s, noise, noise_s = specs(0, 0, 20, 4, 0)
    mbar, vbar = cotangents(4, 1)
    got = pmv.post_mean_var_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, mbar, vbar)
    assert np.all(np.isfinite(got["xs"])) and np.all(np.isfinite(got["x"]))
    if family == cr.MATERN12:
        return
    h = 1e-6

    def f(XX):
        m, v = ref.post_mean_and_var(ref.posterior(k, mean, noise, X, y), XX, mean_s=mean_s, noise_s=noise_s)
        return float(np.dot(mbar, m) + np.dot(vbar, v))
    for d in range(2):
        Xp, Xm = Xs.copy(), Xs.copy()
        Xp[0, d] += h
        Xm[0, d] -= h
        fd = (f(Xp) - f(Xm)) / (2 * h)
        assert abs(got["xs"][0, d] - fd) <= 1e-6 * max(1.0, abs(fd)), (d, got["xs"][0, d], fd)


# ---- the Python mirror through a stand-in library ---------------------------------------------------------------------
class PostMeanVarFakeLib(CompositeFakeLib):
    """answers agp_post_mean_var and agp_post_mean_var_grad from the model and records the arguments"""

    def __init__(self):
        super().__init__()
        self.seen = []

    def _model(self, p, layout, Xs, M, mean_s, noise_s, mba, vba):
        post = self.posts[self._h(p)]
        dt = post["x"].dtype
        X = post["x"].astype(np.float64)
        n, D = X.shape
        Xa = self._points(layout, Xs, M, D, dt).astype(np.float64)
        y = post["delta"] + post["mean"].vector(n, np.float64)
        r = pmv.post_mean_var_grad(post["k"], post["mean"], post["noise"], X, y, Xa, mean_s, noise_s, mba, vba)
        return dt, n, D, Xa, r

    def agp_post_mean_var(self, p, layout, Xs, M, ms, ns, mean_out, var_out):
        dt = self.posts[self._h(p)]["x"].dtype
        mean_s = self._mean(ms, M, dt) if fake_libagp._struct(ms) is not None else self.posts[self._h(p)]["mean"]
        noise_s = self._noise(ns, M, dt) if fake_libagp._struct(ns) is not None else ref.NoiseSpec(0, 0.0)
        _, _, _, _, r = self._model(p, layout, Xs, M, mean_s, noise_s, np.zeros(M), np.zeros(M))
        fake_libagp._arr(mean_out, (M,), dt)[...] = r["mean"]
        fake_libagp._arr(var_out, (M,), dt)[...] = r["var"]
        return 0

    def agp_post_mean_var_grad(self, p, layout, Xs, M, mb, vb, g, nd, md, yb, xg, xsg):
        if fake_libagp._addr(Xs) is None or layout not in (0, 1):
            return self._fail(fake_libagp.INVALID, "invalid")
        if M < 1:
            return self._fail(fake_libagp.DIM, "M")
        dt = self.posts[self._h(p)]["x"].dtype
        addr = lambda q: q is not None and fake_libagp._addr(q) is not None  # noqa: E731
        mba = np.array(fake_libagp._arr(mb, (M,), dt), dtype=np.float64) if addr(mb) else np.zeros(M)
        vba = np.array(fake_libagp._arr(vb, (M,), dt), dtype=np.float64) if addr(vb) else np.zeros(M)
        # the test mean and noise enter the values only, which this call does not return
        dt, n, D, Xa, r = self._model(p, layout, Xs, M, ref.MeanSpec(), ref.NoiseSpec(0, 1e-18), mba, vba)
        self.seen.append(dict(layout=layout, Xs=Xa.copy(), mb=mba.copy() if addr(mb) else None,
                              vb=vba.copy() if addr(vb) else None, outs=(g is not None,) + tuple(addr(q) for q in (nd, md, yb, xg, xsg))))
        if g is not None:
            np.ctypeslib.as_array(g, shape=(len(r["grad"]),))[:] = r["grad"]
        for q, v in [(nd, r["noise_diag"]), (md, r["mean_diag"]), (yb, r["y"])]:
            if addr(q):
                fake_libagp._arr(q, (n,), dt)[...] = v
        for q, v, m in [(xg, r["x"], n), (xsg, r["xs"], M)]:  # in the input layout
            if addr(q):
                fake_libagp._arr(q, (m, D), dt, "C" if layout == 0 else "F")[...] = v
        return 0


@pytest.fixture()
def fake_ag(ag, monkeypatch):
    eng = ag.api.Engine.__new__(ag.api.Engine)
    lib = PostMeanVarFakeLib()
    eng.L, eng.h, eng.device = lib, C.c_void_p(1), 0
    monkeypatch.setattr(ag.api, "_engine", eng)
    return ag, lib


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("container", ["row", "col", "vec"])
def test_python_mirror_passes_the_arguments(fake_ag, dtype, container):
    ag, lib = fake_ag
    D = 1 if container == "vec" else 2
    N, M = 20, 9
    X, y, Xs, _ = problem(N, M, D, 1, seed=1)
    mb, vb = cotangents(M, 1)
    X, y, Xs, mb, vb = X.astype(dtype), y.astype(dtype), Xs.astype(dtype), mb.astype(dtype), vb.astype(dtype)
    wrap = {"row": lambda A: ag.RowVecs(A), "col": lambda A: ag.ColVecs(A.T.copy()), "vec": lambda A: A[:, 0].copy()}[container]
    k = 1.3 * ag.with_lengthscale(ag.SqExponentialKernel(), 1 / 0.7)
    p = ag.posterior(ag.GP(0.3, k)(wrap(X), 0.1), y)
    (mean, var), g = ag.posterior_mean_var_grad(p(wrap(Xs), 0.05), mb, vb, inputs=True)
    seen = lib.seen[-1]
    assert seen["layout"] == 0
    assert seen["outs"] == (True, False, False, True, True, True)
    np.testing.assert_array_equal(seen["mb"], mb.astype(np.float64))
    np.testing.assert_array_equal(seen["vb"], vb.astype(np.float64))
    np.testing.assert_array_equal(seen["Xs"], Xs.astype(np.float64))
    X64, Xs64 = X.astype(np.float64), Xs.astype(np.float64)
    want = pmv.post_mean_var_grad(ref.KernelSpec(cr.SE, 1.3, cr.T_SCALE, 0.7), ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1),
                                  X64, y.astype(np.float64), Xs64, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.05),
                                  mb.astype(np.float64), vb.astype(np.float64))
    tol = 1e-9 if dtype == np.float64 else 1e-4
    assert mean.shape == (M,) and var.shape == (M,) and mean.dtype == dtype
    np.testing.assert_allclose(mean, want["mean"], rtol=tol, atol=tol)
    np.testing.assert_allclose(var, want["var"], rtol=tol, atol=tol)  # the test noise is in the variances
    assert set(g) == {"variance", "scale", "noise", "mean_c", "y", "noise_s", "x", "xs"}
    shp = lambda n: {"row": (n, D), "col": (D, n), "vec": (n,)}[container]  # noqa: E731
    assert g["x"].shape == shp(N) and g["xs"].shape == shp(M) and g["xs"].dtype == dtype
    for key, i in [("variance", 0), ("scale", 1), ("noise", 3), ("mean_c", 4)]:
        np.testing.assert_allclose(g[key], want["grad"][i], rtol=tol)
    np.testing.assert_allclose(g["noise_s"], np.sum(vb.astype(np.float64)), rtol=1e-12)
    np.testing.assert_allclose(g["y"], want["y"], rtol=tol, atol=tol * np.abs(want["y"]).max())
    back = {"row": lambda a: a, "col": lambda a: a.T, "vec": lambda a: a[:, None]}[container]
    for key in ("x", "xs"):
        np.testing.assert_allclose(back(g[key]), want[key], rtol=tol, atol=tol * np.abs(want[key]).max())


def test_python_mirror_test_side_only(fake_ag):
    """training=False passes NULL for every training-side output and returns the test side only; None cotangents are
    NULL; per-point noises and a CustomMean; errors"""
    ag, lib = fake_ag
    N, M, D = 18, 7, 2
    X, y, Xs, _ = problem(N, M, D, 1, seed=3)
    mb, vb = cotangents(M, 3)
    s2, s2s = np.full(N, 0.1), np.linspace(0.02, 0.08, M)
    p = ag.posterior(ag.GP(ag.CustomMean(lambda x: np.sin(x[0])), ag.Matern52Kernel())(ag.RowVecs(X), s2), y)
    fx = p(ag.RowVecs(Xs), s2s)
    _, g = ag.posterior_mean_var_grad(fx, mb, vb, inputs=True, training=False)
    seen = lib.seen[-1]
    assert seen["outs"] == (False, False, False, False, False, True)
    assert set(g) == {"noise_s", "mean_s_v", "xs"}
    want = pmv.post_mean_var_grad(ref.KernelSpec(cr.MATERN52), ref.MeanSpec(2, v=np.sin(X[:, 0])), ref.NoiseSpec(1, v=s2), X,
                                  y, Xs, ref.MeanSpec(2, v=np.sin(Xs[:, 0])), ref.NoiseSpec(1, v=s2s), mb, vb)
    np.testing.assert_allclose(g["xs"], want["xs"], rtol=1e-12, atol=1e-12)
    np.testing.assert_array_equal(g["noise_s"], vb)
    np.testing.assert_array_equal(g["mean_s_v"], mb)
    _, g = ag.posterior_mean_var_grad(fx, None, vb)  # training side, no inputs
    seen = lib.seen[-1]
    assert seen["mb"] is None and seen["outs"] == (True, True, True, True, False, False)
    assert set(g) == {"variance", "noise", "mean_v", "y", "noise_s", "mean_s_v"}
    np.testing.assert_array_equal(g["mean_s_v"], np.zeros(M))
    with pytest.raises(ag.DimensionMismatch):
        ag.posterior_mean_var_grad(fx, mb[:-1], vb)
    with pytest.raises(ag.AGPError):  # a FiniteGP over the prior has no posterior handle
        ag.posterior_mean_var_grad(ag.GP(ag.Matern52Kernel())(ag.RowVecs(X), s2), np.ones(N), np.ones(N))


def test_python_mirror_composite(fake_ag):
    """every kernel parameter's cotangent against central differences of the model's means and variances over refits"""
    ag, lib = fake_ag
    D, N, M = 1, 24, 8
    X, y, Xs, _ = problem(N, M, D, 1, seed=2)
    mb, vb = cotangents(M, 2)
    k = 0.8 * ag.with_lengthscale(ag.SqExponentialKernel(), 2.0) + 0.5 * ag.LinearKernel(c=0.4)
    p = ag.posterior(ag.GP(k)(X[:, 0], 0.1), y)
    _, g = ag.posterior_mean_var_grad(p(Xs[:, 0], 0.05), mb, vb)
    assert len(g["kernel"]) == len(ag.kernel_params(k))
    h = 1e-6
    vals = ag.kernel_params(k)

    def F(vv):
        kc = cr.from_struct(ag.api._kernel_struct(ag.with_kernel_params(k, vv), np.float64, [], D=D), D, np.float64)
        r = pmv.post_mean_var_grad(kc, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, y, Xs, ref.MeanSpec(), ref.NoiseSpec(0, 0.05),
                                   mb, vb)
        return float(np.dot(mb, r["mean"]) + np.dot(vb, r["var"]))
    for i in range(len(vals)):
        vp, vm = list(vals), list(vals)
        vp[i], vm[i] = vals[i] + h, vals[i] - h
        fd = (F(vp) - F(vm)) / (2 * h)
        assert abs(g["kernel"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, g["kernel"][i], fd)


# ---- the C ABI and the Julia rule (the shim cannot be executed here: its structure is held to agp.h) --------------------
def test_cabi_prototype_matches_the_header(ag):
    restype, args = ag._cabi.SIGNATURES["agp_post_mean_var_grad"]
    assert restype is C.c_int32
    assert len(args) == _header_arity("agp_post_mean_var_grad") == 12
    assert [a is C.c_int32 for a in args].count(True) == 1 and args[1] is C.c_int32 and args[3] is C.c_int64
    assert args[6] is not C.c_void_p and args[6]._type_ is C.c_double  # grad_out: double*


RULE_HEAD = ("function CRC.rrule(config::CRC.RuleConfig{>:CRC.HasReverseMode}, ::typeof(mean_and_var), "
             "fx::DevPostFiniteGP{T}) where {T}")
PULLBACK_HEAD = "function post_mean_var_rrule(fx::DevPostFiniteGP{T}, zero_mean::Bool) where {T}"


def test_julia_ccall_arity():
    """the argument-type tuple of the shim's ccall has one entry per parameter of the C prototype, and as many values"""
    src = _julia()
    head = "ccall((:agp_post_mean_var_grad, libagp), Int32,"
    assert src.count(head) == 1
    i = src.index("(", src.index(head) + len(head))
    depth, commas, j = 0, 0, i
    while True:
        ch = src[j]
        depth += ch in "({"
        depth -= ch in ")}"
        commas += ch == "," and depth == 1
        if depth == 0:
            break
        j += 1
    assert commas + 1 == _header_arity("agp_post_mean_var_grad"), src[i:j + 1]
    rest = src[j + 1:src.index("))", j)]
    assert rest.count(",") - 1 == _header_arity("agp_post_mean_var_grad") - 1, rest


def test_julia_rule_forward_is_the_primal():
    """the primal method and the rule compute the means and variances through the same function; one device call with
    every output in the pullback"""
    src = _julia()
    assert src.count(RULE_HEAD) == 1
    assert ("mean_and_var(fx::FiniteGP{<:DevPosterior,<:DevInputs{T},<:Diagonal}) where {T} = "
            "post_mean_var_primal(fx, false)") in src
    body = _rule(src, PULLBACK_HEAD)
    assert "post_mean_var_primal(fx, zero_mean)" in body
    assert body.count("ccall((:agp_post_mean_var_grad, libagp)") == 1
    assert "p.data.C.h, layout, Xs, M, m̄, v̄, g, nd, C_NULL, ȳ, xg, xsg" in body
    assert "Δ isa CRC.AbstractZero && return" in body
    for helper in ("kernel_tangent(", "composite_grads(", "mean_tangent(", "noise_tangent(", "x_tangent(", "as_storage("):
        assert helper in body, helper
    assert "C=(noise=g[4], noise_diag=nd)" in body and "δ=ȳ" in body
    assert "Σy=noise_tangent(fx.Σy, (noise=sum(v̄), noise_diag=v̄))" in body
    assert "return CRC.NoTangent(), f̄x" in body


def test_julia_rule_splits_a_custom_mean():
    """a CustomMean prior goes through AD of the closure's values at x* plus a zero-test-mean device call"""
    src = _julia()
    rule = _rule(src, RULE_HEAD)
    assert ("fx.f.prior.mean isa AbstractGPs.CustomMean && "
            "return CRC.rrule_via_ad(config, mean_split_post_mean_var, fx)") in rule
    split = _rule(src, "function mean_split_post_mean_var(fx::DevPostFiniteGP{T}) where {T}")
    assert "AbstractGPs.mean_vector(fx.f.prior.mean, fx.x)" in split and "zero_mean_post_mean_var(fx)" in split
    assert "mean_spec(AbstractGPs.ZeroMean(), fx.x, T)" in _rule(src, "function post_mean_var_primal(")
    assert ("CRC.rrule(::typeof(zero_mean_post_mean_var), fx::DevPostFiniteGP) = post_mean_var_rrule(fx, true)"
            in src)


def test_julia_tangents_name_only_primal_fields():
    found = _tangent_fields(_rule(_julia(), PULLBACK_HEAD))
    assert len(found) == 4
    for primal, names in found:
        assert primal in PRIMAL_FIELDS, primal
        assert names and set(names) <= PRIMAL_FIELDS[primal], (primal, names)
