"""The gradient of the held-out log-likelihood logpdf(posterior(fx, y)(x*, Sigma*), Y*) (agp_post_pred_logpdf_grad)
without a GPU: the NumPy model tests/pred_logpdf_grad_ref.py pinned to torch fp64 autograd through torch.linalg.cholesky
of both C and Sigma, with every hyper-parameter, both noises, both means, both input sets, y and Y* as leaves; y and Y*
by central differences; the value against the oracle; the Python mirror's argument passing through a stand-in library;
and the structure and ccall arity of the two Julia rules."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import composite_ref as cr
import fake_libagp
import pred_logpdf_grad_ref as pr
from oracle import agp_ref as ref
from test_api_composite_fake import CompositeFakeLib
from test_grad_x_model import mauna_loa_shape
from test_rand_grad_model import _leaf, _torch_factor, single
import grad_x_ref as gx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]
RTOL = 1e-10


def torch_pullback(k, mean, mean_s, noise, noise_s, X, y, Xs, Ys, w):
    """autograd of sum_s w_s logpdf(posterior(fx, y)(x*, Sigma*), Y*[:, s]): (value, descriptor-order kernel gradient,
    training noise, mean, x, y, test noise, mean, x*, Y*); a constant mean is one leaf shared by both sides"""
    torch = pytest.importorskip("torch")
    kc = gx.as_composite(k)
    N, M = X.shape[0], Xs.shape[0]
    Xt, Xst, yt, Yt = _leaf(torch, X), _leaf(torch, Xs), _leaf(torch, y), _leaf(torch, Ys)
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
    Sig = Kss - A.T @ A + torch.diag(s2s * torch.ones(M, dtype=torch.float64))
    Ls = torch.linalg.cholesky(Sig)
    Zq = torch.linalg.solve_triangular(Ls, Yt - mu[:, None], upper=False)
    lp = -0.5 * (M * math.log(2 * math.pi) + 2.0 * torch.log(torch.diagonal(Ls)).sum() + (Zq * Zq).sum(0))
    (lp * torch.as_tensor(np.asarray(w, dtype=np.float64))).sum().backward()
    kg = np.concatenate([np.atleast_1d(t.grad.numpy()) for t in leaves])
    g = lambda t: None if t.grad is None else t.grad.numpy()  # noqa: E731
    return (lp.detach().numpy(), kg, g(s2), g(mt), Xt.grad.numpy(), yt.grad.numpy(), g(s2s), g(mst), Xst.grad.numpy(),
            Yt.grad.numpy())


def problem(N, M, D, S, seed=0):
    rng = np.random.default_rng(seed + 13 * N + 7 * M + 5 * D + S)
    return rng.uniform(-2, 2, (N, D)), rng.standard_normal(N), rng.uniform(-2.5, 2.5, (M, D)), rng.standard_normal((M, S))


def weights(S, kind):
    """all ones, or mixed signs with a zero"""
    if kind == "ones":
        return np.ones(S)
    w = np.random.default_rng(S).uniform(-1.5, 2.0, S)
    w[S // 2] = 0.0
    return w


def close(a, b, rtol=RTOL):
    b = np.asarray(b, dtype=np.float64)
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * max(1.0, np.abs(b).max()))


def specs(mean_kind, noise_kind, N, M, seed):
    rng = np.random.default_rng(seed)
    mean = [ref.MeanSpec(), ref.MeanSpec(1, 0.3), ref.MeanSpec(2, v=rng.standard_normal(N))][mean_kind]
    mean_s = [ref.MeanSpec(), ref.MeanSpec(1, 0.3), ref.MeanSpec(2, v=rng.standard_normal(M))][mean_kind]
    noise = ref.NoiseSpec(0, 0.1) if noise_kind == 0 else ref.NoiseSpec(1, v=rng.uniform(0.05, 0.2, N))
    noise_s = ref.NoiseSpec(0, 0.05) if noise_kind == 0 else ref.NoiseSpec(1, v=rng.uniform(0.02, 0.2, M))
    return mean, mean_s, noise, noise_s


def _check(k, mean, mean_s, noise, noise_s, X, y, Xs, Ys, w):
    got = pr.pred_logpdf_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, Ys, w)
    lp, kg, ng, mg, xg, yg, nsg, msg, xsg, Yg = torch_pullback(k, mean, mean_s, noise, noise_s, X, y, Xs, Ys, w)
    close(got["lp"], lp)
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
    close(got["Ys"], Yg)


@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_model_matches_torch_autograd(family, transform):
    D = 3
    k = single(family, transform, D, np.random.default_rng(family + 3 * transform))
    for S in (1, 3, 130):
        for wkind in ("ones", "mixed"):
            for noise_kind in (0, 1):
                for mean_kind in (0, 1, 2):
                    N, M = 24 + 2 * mean_kind + noise_kind, 11 + mean_kind
                    X, y, Xs, Ys = problem(N, M, D, S, seed=family + mean_kind)
                    if family == cr.LINEAR:  # a rank-D kernel: shorter inputs keep Sigma's conditioning near the others'
                        X, Xs = 0.5 * X, 0.5 * Xs
                    mean, mean_s, noise, noise_s = specs(mean_kind, noise_kind, N, M, mean_kind + 3 * noise_kind)
                    _check(k, mean, mean_s, noise, noise_s, X, y, Xs, Ys, weights(S, wkind))


@pytest.mark.parametrize("D", [1, 3])
def test_model_matches_torch_autograd_mauna_loa(D):
    X, y, Xs, Ys = problem(30, 12, D, 3, seed=6)
    mean, mean_s, noise, noise_s = specs(2, 1, 30, 12, D)
    _check(mauna_loa_shape(D, np.random.default_rng(D)), mean, mean_s, noise, noise_s, X, y, Xs, Ys, weights(3, "mixed"))


def test_y_and_ys_match_central_differences():
    """ybar and Ybar* against central differences of the oracle's own held-out logpdf over refits"""
    k = single(cr.MATERN32, cr.T_ARD, 2, np.random.default_rng(0))
    X, y, Xs, Ys = problem(25, 9, 2, 4, seed=9)
    mean, mean_s, noise, noise_s = specs(1, 0, 25, 9, 1)
    w = weights(4, "mixed")
    got = pr.pred_logpdf_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, Ys, w)

    def f(yy, YY):
        return float(np.dot(w, ref.post_logpdf(ref.posterior(k, mean, noise, X, yy), Xs, noise_s, YY, mean_s)))
    h = 1e-6
    for i in (0, 7, 24):
        yp, ym = y.copy(), y.copy()
        yp[i] += h
        ym[i] -= h
        fd = (f(yp, Ys) - f(ym, Ys)) / (2 * h)
        assert abs(got["y"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, got["y"][i], fd)
    for i, s in [(0, 0), (4, 1), (8, 3)]:
        Yp, Ym = Ys.copy(), Ys.copy()
        Yp[i, s] += h
        Ym[i, s] -= h
        fd = (f(y, Yp) - f(y, Ym)) / (2 * h)
        assert abs(got["Ys"][i, s] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, s, got["Ys"][i, s], fd)


@pytest.mark.parametrize("kname", ["single", "mauna_loa"])
def test_value_matches_the_oracle(kname):
    rng = np.random.default_rng(3)
    X, y, Xs, Ys = problem(28, 10, 2, 5, seed=4)
    if kname == "single":
        k = single(cr.SE, cr.T_SCALE, 2, rng)
        mean, mean_s, noise, noise_s = specs(2, 1, 28, 10, 5)
        want = ref.post_logpdf(ref.posterior(k, mean, noise, X, y), Xs, noise_s, Ys, mean_s)
    else:  # composite_ref's posterior carries its own (constant) mean to x*
        k = mauna_loa_shape(2, rng)
        mean, mean_s, noise, noise_s = specs(1, 1, 28, 10, 5)
        want = cr.post_logpdf(cr.posterior(k, mean, noise, X, y), Xs, noise_s, Ys)
    got = pr.pred_logpdf_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, Ys)
    close(got["lp"], want, 1e-11)


# ---- the Python mirror through a stand-in library ---------------------------------------------------------------------
class PredFakeLib(CompositeFakeLib):
    """answers agp_post_pred_logpdf_grad from the model and records the arguments"""

    def __init__(self):
        super().__init__()
        self.seen = []

    def agp_post_pred_logpdf_grad(self, p, layout, Xs, M, ms, ns, Ys, S, lp_bar, lp_out, g, nd, md, yb, xg, nsd, msd, ysb,
                                  xsg):
        post = self.posts[self._h(p)]
        dt = post["x"].dtype
        X = post["x"].astype(np.float64)
        n, D = X.shape
        if S < 1 or fake_libagp._addr(Ys) is None or layout not in (0, 1):
            return self._fail(fake_libagp.INVALID, "invalid")
        Xa = self._points(layout, Xs, M, D, dt).astype(np.float64)
        mean_s = self._mean(ms, M, dt) if fake_libagp._struct(ms) is not None else post["mean"]
        noise_s = self._noise(ns, M, dt) if fake_libagp._struct(ns) is not None else ref.NoiseSpec(0, 1e-18)
        Ya = np.array(fake_libagp._arr(Ys, (M, S), dt, "F"), dtype=np.float64)
        w = np.ones(S) if not lp_bar else np.array(np.ctypeslib.as_array(lp_bar, shape=(S,)))
        addr = lambda q: fake_libagp._addr(q) is not None  # noqa: E731
        self.seen.append(dict(S=S, w=None if not lp_bar else w.copy(), layout=layout, Ys=Ya.copy(), Xs=Xa.copy(),
                              mean_s=mean_s, noise_s=noise_s, outs=tuple(addr(q) for q in (nd, md, yb, xg, nsd, msd, ysb, xsg))))
        y = post["delta"] + post["mean"].vector(n, np.float64)
        r = pr.pred_logpdf_grad(post["k"], post["mean"], post["noise"], X, y, Xa, mean_s, noise_s, Ya, w)
        fake_libagp._arr(lp_out, (S,), dt)[...] = r["lp"]
        np.ctypeslib.as_array(g, shape=(len(r["grad"]),))[:] = r["grad"]
        for q, v, shape in [(nd, r["noise_diag"], (n,)), (md, r["mean_diag"], (n,)), (yb, r["y"], (n,)),
                            (nsd, r["noise_s_diag"], (M,)), (msd, r["mean_s_diag"], (M,)), (ysb, r["Ys"], (M, S))]:
            if addr(q):
                fake_libagp._arr(q, shape, dt, "F")[...] = v
        for q, v, m in [(xg, r["x"], n), (xsg, r["xs"], M)]:  # in the input layout
            if addr(q):
                if layout == 0:
                    fake_libagp._arr(q, (m, D), dt)[...] = v
                else:
                    fake_libagp._arr(q, (m, D), dt, "F")[...] = v
        return 0


@pytest.fixture()
def fake_ag(ag, monkeypatch):
    eng = ag.api.Engine.__new__(ag.api.Engine)
    lib = PredFakeLib()
    eng.L, eng.h, eng.device = lib, C.c_void_p(1), 0
    monkeypatch.setattr(ag.api, "_engine", eng)
    return ag, lib


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("container", ["row", "col", "vec"])
def test_python_mirror_passes_the_arguments(fake_ag, dtype, container):
    ag, lib = fake_ag
    D = 1 if container == "vec" else 2
    N, M, S = 20, 9, 3
    X, y, Xs, Ys = problem(N, M, D, S, seed=1)
    X, y, Xs, Ys = X.astype(dtype), y.astype(dtype), Xs.astype(dtype), Ys.astype(dtype)
    wrap = {"row": lambda A: ag.RowVecs(A), "col": lambda A: ag.ColVecs(A.T.copy()), "vec": lambda A: A[:, 0].copy()}[container]
    k = 1.3 * ag.with_lengthscale(ag.SqExponentialKernel(), 1 / 0.7)
    p = ag.posterior(ag.GP(0.3, k)(wrap(X), 0.1), y)
    lp, g = ag.posterior_logpdf_grad(p(wrap(Xs), 0.05), Ys, inputs=True)
    seen = lib.seen[-1]
    assert (seen["S"], seen["w"], seen["layout"]) == (S, None, 0)  # lp_bar=None -> NULL (all ones)
    assert seen["outs"] == (False, False, True, True, True, False, True, True)
    np.testing.assert_array_equal(seen["Ys"], Ys.astype(np.float64))
    np.testing.assert_array_equal(seen["Xs"], Xs.astype(np.float64))
    X64, Xs64 = X.astype(np.float64), Xs.astype(np.float64)
    want = pr.pred_logpdf_grad(ref.KernelSpec(cr.SE, 1.3, cr.T_SCALE, 0.7), ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X64,
                               y.astype(np.float64), Xs64, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.05), Ys.astype(np.float64))
    tol = 1e-9 if dtype == np.float64 else 1e-4
    assert lp.shape == (S,) and lp.dtype == dtype
    assert set(g) == {"variance", "scale", "noise", "mean_c", "y", "noise_s", "Y", "x", "xs"}
    assert g["Y"].shape == (M, S) and g["Y"].dtype == dtype and g["y"].shape == (N,)
    shp = lambda n: {"row": (n, D), "col": (D, n), "vec": (n,)}[container]  # noqa: E731
    assert g["x"].shape == shp(N) and g["xs"].shape == shp(M) and g["x"].dtype == dtype
    for key, i in [("variance", 0), ("scale", 1), ("noise", 3), ("mean_c", 4)]:
        np.testing.assert_allclose(g[key], want["grad"][i], rtol=tol)
    np.testing.assert_allclose(g["noise_s"], np.sum(want["noise_s_diag"]), rtol=tol)
    for key, wk in [("Y", "Ys"), ("y", "y")]:
        np.testing.assert_allclose(g[key], want[wk], rtol=tol, atol=tol * np.abs(want[wk]).max())
    back = {"row": lambda a: a, "col": lambda a: a.T, "vec": lambda a: a[:, None]}[container]
    for key in ("x", "xs"):
        np.testing.assert_allclose(back(g[key]), want[key], rtol=tol, atol=tol * np.abs(want[key]).max())
    np.testing.assert_allclose(lp, want["lp"], rtol=tol)


def test_python_mirror_weights_vector_y_custom_mean(fake_ag):
    """lp_bar reaches the call; a vector Y is one column; a CustomMean's values at x* are passed; per-point noises"""
    ag, lib = fake_ag
    N, M, D = 18, 7, 2
    X, y, Xs, Ys = problem(N, M, D, 1, seed=3)
    s2, s2s = np.full(N, 0.1), np.linspace(0.02, 0.08, M)
    mf = lambda x: np.sin(x[0])  # noqa: E731
    p = ag.posterior(ag.GP(ag.CustomMean(mf), ag.Matern52Kernel())(ag.RowVecs(X), s2), y)
    lp, g = ag.posterior_logpdf_grad(p(ag.RowVecs(Xs), s2s), Ys[:, 0], lp_bar=[-0.5])
    seen = lib.seen[-1]
    assert seen["S"] == 1 and list(seen["w"]) == [-0.5] and seen["outs"][:2] == (True, True) and not seen["outs"][3]
    np.testing.assert_allclose(seen["mean_s"].v, np.sin(Xs[:, 0]), rtol=1e-15)
    want = pr.pred_logpdf_grad(ref.KernelSpec(cr.MATERN52), ref.MeanSpec(2, v=np.sin(X[:, 0])), ref.NoiseSpec(1, v=s2), X, y,
                               Xs, ref.MeanSpec(2, v=np.sin(Xs[:, 0])), ref.NoiseSpec(1, v=s2s), Ys, [-0.5])
    assert np.ndim(lp) == 0 and g["Y"].shape == (M,) and g["noise"].shape == (N,) and g["noise_s"].shape == (M,)
    assert "x" not in g and "xs" not in g
    for key, wk in [("mean_v", "mean_diag"), ("mean_s_v", "mean_s_diag"), ("noise", "noise_diag"),
                    ("noise_s", "noise_s_diag"), ("y", "y")]:
        np.testing.assert_allclose(g[key], want[wk], rtol=1e-12)
    np.testing.assert_allclose(g["Y"], want["Ys"][:, 0], rtol=1e-12)
    with pytest.raises(ag.DimensionMismatch):
        ag.posterior_logpdf_grad(p(ag.RowVecs(Xs), s2s), Ys[:, 0], lp_bar=[1.0, 2.0])
    with pytest.raises(ag.DimensionMismatch):
        ag.posterior_logpdf_grad(p(ag.RowVecs(Xs), s2s), Ys[:-1, 0])
    with pytest.raises(ag.AGPError):  # a FiniteGP over the prior is not this function's
        ag.posterior_logpdf_grad(ag.GP(ag.Matern52Kernel())(ag.RowVecs(X), s2), y)


def test_python_mirror_composite(fake_ag):
    """every kernel parameter's cotangent against central differences of the held-out logpdf over refits"""
    ag, lib = fake_ag
    D, N, M, S = 1, 24, 8, 3
    X, y, Xs, Ys = problem(N, M, D, S, seed=2)
    k = 0.8 * ag.with_lengthscale(ag.SqExponentialKernel(), 2.0) + 0.5 * ag.RationalQuadraticKernel(alpha=1.3)
    w = np.array([1.0, -0.3, 2.0])
    p = ag.posterior(ag.GP(k)(X[:, 0], 0.1), y)
    lp, g = ag.posterior_logpdf_grad(p(Xs[:, 0], 0.05), Ys, lp_bar=w)
    assert len(g["kernel"]) == len(ag.kernel_params(k))
    h = 1e-6
    vals = ag.kernel_params(k)

    def F(vv):
        kc = cr.from_struct(ag.api._kernel_struct(ag.with_kernel_params(k, vv), np.float64, [], D=D), D, np.float64)
        return float(np.dot(w, pr.pred_logpdf_grad(kc, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, y, Xs, ref.MeanSpec(),
                                                   ref.NoiseSpec(0, 0.05), Ys)["lp"]))
    for i in range(len(vals)):
        vp, vm = list(vals), list(vals)
        vp[i], vm[i] = vals[i] + h, vals[i] - h
        fd = (F(vp) - F(vm)) / (2 * h)
        assert abs(g["kernel"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, g["kernel"][i], fd)


# ---- the C ABI and the Julia rules (the shim cannot be executed here: its structure is held to agp.h) -------------------
def _header_arity(name):
    src = open(os.path.join(ROOT, "include", "agp.h")).read()
    a = src.index("int32_t %s(" % name)
    return src[a:src.index(";", a)].count(",") + 1


def test_cabi_prototype_matches_the_header(ag):
    restype, args = ag._cabi.SIGNATURES["agp_post_pred_logpdf_grad"]
    assert len(args) == _header_arity("agp_post_pred_logpdf_grad") == 19


def _julia():
    return open(os.path.join(ROOT, "julia", "AGPBlackwell.jl")).read()


def _rule(src, head):
    a = src.index(head)
    return src[a:src.index("\nend\n", a)]


def test_julia_ccall_arity():
    """the argument-type tuple of the shim's ccall has one entry per parameter of the C prototype"""
    src = _julia()
    a = src.index("ccall((:agp_post_pred_logpdf_grad, libagp), Int32,")
    i = src.index("(", a + len("ccall((:agp_post_pred_logpdf_grad, libagp), Int32,"))
    depth, commas, j = 0, 0, i
    while True:
        ch = src[j]
        depth += ch in "({"
        depth -= ch in ")}"
        commas += ch == "," and depth == 1
        if depth == 0:
            break
        j += 1
    assert commas + 1 == _header_arity("agp_post_pred_logpdf_grad"), src[i:j + 1]
    # the values passed: the same count after the tuple
    rest = src[j + 1:src.index("))", j)]
    assert rest.count(",") - 1 == _header_arity("agp_post_pred_logpdf_grad") - 1, rest


POSTERIOR_HEAD = "function CRC.rrule(::typeof(posterior), fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}"
PRED_HEAD = "function CRC.rrule(::typeof(logpdf), fx::DevPostFiniteGP{T}, Y::AbstractVecOrMat{<:Real}) where {T}"


def test_julia_posterior_rule():
    src = _julia()
    rule = _rule(src, POSTERIOR_HEAD)
    assert rule.split("\n")[1].strip().startswith("claimed(fx.f) || return nothing")
    assert "post = posterior(fx, y)" in rule
    # the tangent of the DevPosterior is re-routed: prior -> fx.f, data.x -> fx.x, data.δ -> y and the mean,
    # data.C -> fx.Σy
    for piece in ("Δp.prior", "Δd.x", "Δd.δ", "noise_tangent(fx.Σy, Δd.C)", "mean_tangent(", "tangent_c(Δf.mean)", ") - sum(ȳ)"):
        assert piece in rule, piece
    # no sum of a tangent handed in by the AD system with one built here
    assert "Δf.mean +" not in rule and "+ mean_tangent" not in rule
    assert "return CRC.NoTangent(), f̄x, ȳ" in rule


def test_julia_pred_logpdf_rule():
    src = _julia()
    rule = _rule(src, PRED_HEAD)
    assert rule.count("ccall((:agp_post_pred_logpdf_grad, libagp)") == 1
    assert "w = convert(Vector{Float64}, Δ isa Real ? [Δ] : Δ)" in rule
    for helper in ("kernel_tangent(", "composite_grads(", "mean_tangent(", "noise_tangent(", "x_tangent("):
        assert helper in rule, helper
    assert "return CRC.NoTangent(), f̄x, Y isa AbstractVector ? vec(Ȳ) : Ȳ" in rule
    # the training-noise gradient rides in data.C (the diagonal of C's cotangent), which the posterior rule routes to
    # fx.Σy; δ carries ȳ
    assert "C=(noise=g[4], noise_diag=nd)" in rule and "δ=ȳ" in rule
    # the prior logpdf rules are still there
    assert "function CRC.rrule(::typeof(logpdf), fx::DevFiniteGP{T}, Y::AbstractMatrix{<:Real}) where {T}" in src


# the fields of each primal a Tangent is built for in the two rules (AbstractGPs' FiniteGP, GP and PosteriorGP, and the
# NamedTuple the shim stores as a PosteriorGP's data)
PRIMAL_FIELDS = {"fx": {"f", "x", "Σy"}, "fx.f": {"mean", "kernel"}, "p": {"prior", "data"}, "p.prior": {"mean", "kernel"},
                 "p.data": {"α", "C", "x", "δ"}}


def _tangent_fields(rule):
    """(primal expression, top-level keyword names) of every CRC.Tangent{typeof(v)}(; ...) in `rule`"""
    out = []
    head = "CRC.Tangent{typeof("
    i = rule.find(head)
    while i >= 0:
        j = rule.index(")}(", i)
        primal = rule[i + len(head):j]
        k = j + 3
        assert rule[k] == ";", rule[i:i + 80]
        depth, names, start = 1, [], k + 1
        while depth:
            ch = rule[k + 1]
            k += 1
            if ch in "([{":
                depth += 1
            elif ch in ")]}":
                depth -= 1
            if depth == 1 and ch == "=" and rule[k - 1] not in "=<>!" and rule[k + 1] != "=":
                names.append(rule[start:k].strip().split(",")[-1].strip())
            if depth == 1 and ch == ",":
                start = k + 1
        out.append((primal, names))
        i = rule.find(head, k)
    return out


@pytest.mark.parametrize("head", [POSTERIOR_HEAD, PRED_HEAD])
def test_julia_tangents_name_only_primal_fields(head):
    found = _tangent_fields(_rule(_julia(), head))
    assert found
    for primal, names in found:
        assert primal in PRIMAL_FIELDS, primal
        assert names and set(names) <= PRIMAL_FIELDS[primal], (primal, names)
