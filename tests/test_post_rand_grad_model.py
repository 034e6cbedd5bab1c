"""The pullback of rand over an exact posterior (agp_post_rand_grad) without a GPU: the NumPy model
tests/post_rand_grad_ref.py pinned to torch fp64 autograd through torch.linalg.cholesky of both C and Sigma, with every
hyper-parameter, both noises, both means, both input sets, y and Z as leaves; y, x* and Z by central differences; the
Python mirror's argument passing through a stand-in library; and the structure and ccall arity of the Julia rule."""
import ctypes as C
import os

import numpy as np
import pytest

import composite_ref as cr
import fake_libagp
import grad_x_ref as gx
import post_rand_grad_ref as prr
from oracle import agp_ref as ref
from test_api_composite_fake import CompositeFakeLib
from test_grad_x_model import mauna_loa_shape
from test_pred_logpdf_grad_model import (PRIMAL_FIELDS, _header_arity, _julia, _rule, _tangent_fields, close, problem,
                                         specs)
from test_rand_grad_model import _leaf, _torch_factor, single

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]


def torch_pullback(k, mean, mean_s, noise, noise_s, X, y, Xs, Z, Obar):
    """autograd of sum(Obar o (mu* 1' + L* Z)) over posterior(fx, y)(x*, Sigma*): (samples, descriptor-order kernel
    gradient, training noise, mean, x, y, test noise, mean, x*, Z); a constant mean is one leaf shared by both sides"""
    torch = pytest.importorskip("torch")
    kc = gx.as_composite(k)
    N, M = X.shape[0], Xs.shape[0]
    Xt, Xst, yt, Zt = _leaf(torch, X), _leaf(torch, Xs), _leaf(torch, y), _leaf(torch, Z)
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
    Ls = torch.linalg.cholesky(Kss - A.T @ A + torch.diag(s2s * torch.ones(M, dtype=torch.float64)))
    out = mu[:, None] + Ls @ Zt
    (out * torch.as_tensor(np.asarray(Obar, dtype=np.float64))).sum().backward()
    kg = np.concatenate([np.atleast_1d(t.grad.numpy()) for t in leaves])
    g = lambda t: None if t.grad is None else t.grad.numpy()  # noqa: E731
    return (out.detach().numpy(), kg, g(s2), g(mt), Xt.grad.numpy(), yt.grad.numpy(), g(s2s), g(mst), Xst.grad.numpy(),
            Zt.grad.numpy())


def normals(M, S, seed):
    rng = np.random.default_rng(seed + 31 * M + S)
    return rng.standard_normal((M, S)), rng.standard_normal((M, S))


def _check(k, mean, mean_s, noise, noise_s, X, y, Xs, Z, Obar):
    got = prr.post_rand_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, Z, Obar)
    out, kg, ng, mg, xg, yg, nsg, msg, xsg, Zg = torch_pullback(k, mean, mean_s, noise, noise_s, X, y, Xs, Z, Obar)
    close(got["out"], out)
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
    close(got["Z"], Zg)


@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_model_matches_torch_autograd(family, transform):
    D = 3
    k = single(family, transform, D, np.random.default_rng(family + 3 * transform))
    for S in (1, 3, 130):
        for noise_kind in (0, 1):
            for mean_kind in (0, 1, 2):
                N, M = 24 + 2 * mean_kind + noise_kind, 11 + mean_kind
                X, y, Xs, _ = problem(N, M, D, 1, seed=family + mean_kind)
                if family == cr.LINEAR:  # a rank-D kernel: shorter inputs keep Sigma's conditioning near the others'
                    X, Xs = 0.5 * X, 0.5 * Xs
                mean, mean_s, noise, noise_s = specs(mean_kind, noise_kind, N, M, mean_kind + 3 * noise_kind)
                Z, Obar = normals(M, S, family + noise_kind)
                _check(k, mean, mean_s, noise, noise_s, X, y, Xs, Z, Obar)


@pytest.mark.parametrize("D", [1, 3])
def test_model_matches_torch_autograd_mauna_loa(D):
    X, y, Xs, _ = problem(30, 12, D, 1, seed=6)
    mean, mean_s, noise, noise_s = specs(2, 1, 30, 12, D)
    Z, Obar = normals(12, 3, D)
    _check(mauna_loa_shape(D, np.random.default_rng(D)), mean, mean_s, noise, noise_s, X, y, Xs, Z, Obar)


def test_samples_match_the_oracle():
    """the model's forward is the oracle's posterior rand at the same normals"""
    k = single(cr.SE, cr.T_SCALE, 2, np.random.default_rng(0))
    X, y, Xs, _ = problem(28, 10, 2, 1, seed=4)
    mean, mean_s, noise, noise_s = specs(2, 1, 28, 10, 5)
    Z, Obar = normals(10, 4, 1)
    got = prr.post_rand_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, Z, Obar)
    close(got["out"], ref.post_rand_from_Z(ref.posterior(k, mean, noise, X, y), Xs, noise_s, Z, mean_s), 1e-11)


def test_y_xs_and_z_match_central_differences():
    """ybar, the x* gradient and Zbar against central differences of the oracle's posterior rand over refits"""
    k = single(cr.MATERN52, cr.T_ARD, 2, np.random.default_rng(0))
    X, y, Xs, _ = problem(25, 9, 2, 1, seed=9)
    mean, mean_s, noise, noise_s = specs(1, 0, 25, 9, 1)
    Z, Obar = normals(9, 4, 2)
    got = prr.post_rand_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, Z, Obar)

    def f(yy, XX, ZZ):
        return float(np.sum(Obar * ref.post_rand_from_Z(ref.posterior(k, mean, noise, X, yy), XX, noise_s, ZZ, mean_s)))
    h = 1e-6
    for i in (0, 7, 24):
        yp, ym = y.copy(), y.copy()
        yp[i] += h
        ym[i] -= h
        fd = (f(yp, Xs, Z) - f(ym, Xs, Z)) / (2 * h)
        assert abs(got["y"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, got["y"][i], fd)
    for i, d in [(0, 0), (4, 1), (8, 0)]:
        Xp, Xm = Xs.copy(), Xs.copy()
        Xp[i, d] += h
        Xm[i, d] -= h
        fd = (f(y, Xp, Z) - f(y, Xm, Z)) / (2 * h)
        assert abs(got["xs"][i, d] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, d, got["xs"][i, d], fd)
    for i, s in [(0, 0), (4, 1), (8, 3)]:
        Zp, Zm = Z.copy(), Z.copy()
        Zp[i, s] += h
        Zm[i, s] -= h
        fd = (f(y, Xs, Zp) - f(y, Xs, Zm)) / (2 * h)
        assert abs(got["Z"][i, s] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, s, got["Z"][i, s], fd)


# ---- the Python mirror through a stand-in library ---------------------------------------------------------------------
class PostRandFakeLib(CompositeFakeLib):
    """answers agp_post_rand and agp_post_rand_grad from the model and records the arguments"""

    def __init__(self):
        super().__init__()
        self.seen = []

    def _call(self, p, layout, Xs, M, ms, ns, Z, S, Ob):
        post = self.posts[self._h(p)]
        dt = post["x"].dtype
        X = post["x"].astype(np.float64)
        n, D = X.shape
        Xa = self._points(layout, Xs, M, D, dt).astype(np.float64)
        mean_s = self._mean(ms, M, dt) if fake_libagp._struct(ms) is not None else post["mean"]
        noise_s = self._noise(ns, M, dt) if fake_libagp._struct(ns) is not None else ref.NoiseSpec(0, 1e-18)
        Za = np.array(fake_libagp._arr(Z, (M, S), dt, "F"), dtype=np.float64)
        Oa = np.zeros((M, S)) if Ob is None else np.array(fake_libagp._arr(Ob, (M, S), dt, "F"), dtype=np.float64)
        y = post["delta"] + post["mean"].vector(n, np.float64)
        r = prr.post_rand_grad(post["k"], post["mean"], post["noise"], X, y, Xa, mean_s, noise_s, Za, Oa)
        return post, dt, n, D, Xa, Za, Oa, mean_s, noise_s, r

    def agp_post_rand(self, p, layout, Xs, M, ms, ns, Z, S, out):
        r = self._call(p, layout, Xs, M, ms, ns, Z, S, None)
        dt, r = r[1], r[-1]
        fake_libagp._arr(out, (M, S), dt, "F")[...] = r["out"]
        return 0

    def agp_post_rand_grad(self, p, layout, Xs, M, ms, ns, Z, S, Ob, g, nd, md, yb, xg, nsd, msd, zb, xsg):
        if S < 1 or fake_libagp._addr(Z) is None or fake_libagp._addr(Ob) is None or layout not in (0, 1):
            return self._fail(fake_libagp.INVALID, "invalid")
        post, dt, n, D, Xa, Za, Oa, mean_s, noise_s, r = self._call(p, layout, Xs, M, ms, ns, Z, S, Ob)
        addr = lambda q: fake_libagp._addr(q) is not None  # noqa: E731
        self.seen.append(dict(S=S, layout=layout, Z=Za.copy(), Ob=Oa.copy(), Xs=Xa.copy(), mean_s=mean_s, noise_s=noise_s,
                              outs=tuple(addr(q) for q in (nd, md, yb, xg, nsd, msd, zb, xsg))))
        np.ctypeslib.as_array(g, shape=(len(r["grad"]),))[:] = r["grad"]
        for q, v, shape in [(nd, r["noise_diag"], (n,)), (md, r["mean_diag"], (n,)), (yb, r["y"], (n,)),
                            (nsd, r["noise_s_diag"], (M,)), (msd, r["mean_s_diag"], (M,)), (zb, r["Z"], (M, S))]:
            if addr(q):
                fake_libagp._arr(q, shape, dt, "F")[...] = v
        for q, v, m in [(xg, r["x"], n), (xsg, r["xs"], M)]:  # in the input layout
            if addr(q) and layout == 0:
                fake_libagp._arr(q, (m, D), dt)[...] = v
            elif addr(q):
                fake_libagp._arr(q, (m, D), dt, "F")[...] = v
        return 0


@pytest.fixture()
def fake_ag(ag, monkeypatch):
    eng = ag.api.Engine.__new__(ag.api.Engine)
    lib = PostRandFakeLib()
    eng.L, eng.h, eng.device = lib, C.c_void_p(1), 0
    monkeypatch.setattr(ag.api, "_engine", eng)
    return ag, lib


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("container", ["row", "col", "vec"])
def test_python_mirror_passes_the_arguments(fake_ag, dtype, container):
    ag, lib = fake_ag
    D = 1 if container == "vec" else 2
    N, M, S = 20, 9, 3
    X, y, Xs, _ = problem(N, M, D, 1, seed=1)
    Z, Ob = normals(M, S, 1)
    X, y, Xs, Z, Ob = X.astype(dtype), y.astype(dtype), Xs.astype(dtype), Z.astype(dtype), Ob.astype(dtype)
    wrap = {"row": lambda A: ag.RowVecs(A), "col": lambda A: ag.ColVecs(A.T.copy()), "vec": lambda A: A[:, 0].copy()}[container]
    k = 1.3 * ag.with_lengthscale(ag.SqExponentialKernel(), 1 / 0.7)
    p = ag.posterior(ag.GP(0.3, k)(wrap(X), 0.1), y)
    out, g = ag.posterior_rand_grad(p(wrap(Xs), 0.05), Z, Ob, inputs=True)
    seen = lib.seen[-1]
    assert (seen["S"], seen["layout"]) == (S, 0)
    assert seen["outs"] == (False, False, True, True, True, False, True, True)
    np.testing.assert_array_equal(seen["Z"], Z.astype(np.float64))
    np.testing.assert_array_equal(seen["Ob"], Ob.astype(np.float64))
    np.testing.assert_array_equal(seen["Xs"], Xs.astype(np.float64))
    X64, Xs64 = X.astype(np.float64), Xs.astype(np.float64)
    want = prr.post_rand_grad(ref.KernelSpec(cr.SE, 1.3, cr.T_SCALE, 0.7), ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X64,
                              y.astype(np.float64), Xs64, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.05), Z.astype(np.float64),
                              Ob.astype(np.float64))
    tol = 1e-9 if dtype == np.float64 else 1e-4
    assert out.shape == (M, S) and out.dtype == dtype
    assert set(g) == {"variance", "scale", "noise", "mean_c", "y", "noise_s", "Z", "x", "xs"}
    assert g["Z"].shape == (M, S) and g["Z"].dtype == dtype and g["y"].shape == (N,)
    shp = lambda n: {"row": (n, D), "col": (D, n), "vec": (n,)}[container]  # noqa: E731
    assert g["x"].shape == shp(N) and g["xs"].shape == shp(M) and g["x"].dtype == dtype
    for key, i in [("variance", 0), ("scale", 1), ("noise", 3), ("mean_c", 4)]:
        np.testing.assert_allclose(g[key], want["grad"][i], rtol=tol)
    np.testing.assert_allclose(g["noise_s"], np.sum(want["noise_s_diag"]), rtol=tol)
    for key in ("Z", "y"):
        np.testing.assert_allclose(g[key], want[key], rtol=tol, atol=tol * np.abs(want[key]).max())
    back = {"row": lambda a: a, "col": lambda a: a.T, "vec": lambda a: a[:, None]}[container]
    for key in ("x", "xs"):
        np.testing.assert_allclose(back(g[key]), want[key], rtol=tol, atol=tol * np.abs(want[key]).max())
    np.testing.assert_allclose(out, want["out"], rtol=tol, atol=tol)


def test_python_mirror_vector_z_custom_mean(fake_ag):
    """a vector Z is one column; a CustomMean's values at x* are passed; per-point noises; errors"""
    ag, lib = fake_ag
    N, M, D = 18, 7, 2
    X, y, Xs, _ = problem(N, M, D, 1, seed=3)
    Z, Ob = normals(M, 1, 3)
    s2, s2s = np.full(N, 0.1), np.linspace(0.02, 0.08, M)
    mf = lambda x: np.sin(x[0])  # noqa: E731
    p = ag.posterior(ag.GP(ag.CustomMean(mf), ag.Matern52Kernel())(ag.RowVecs(X), s2), y)
    out, g = ag.posterior_rand_grad(p(ag.RowVecs(Xs), s2s), Z[:, 0], Ob[:, 0])
    seen = lib.seen[-1]
    assert seen["S"] == 1 and seen["outs"][:2] == (True, True) and not seen["outs"][3]
    np.testing.assert_allclose(seen["mean_s"].v, np.sin(Xs[:, 0]), rtol=1e-15)
    want = prr.post_rand_grad(ref.KernelSpec(cr.MATERN52), ref.MeanSpec(2, v=np.sin(X[:, 0])), ref.NoiseSpec(1, v=s2), X, y,
                              Xs, ref.MeanSpec(2, v=np.sin(Xs[:, 0])), ref.NoiseSpec(1, v=s2s), Z, Ob)
    assert out.shape == (M,) and g["Z"].shape == (M,) and g["noise"].shape == (N,) and g["noise_s"].shape == (M,)
    assert "x" not in g and "xs" not in g
    for key, wk in [("mean_v", "mean_diag"), ("mean_s_v", "mean_s_diag"), ("noise", "noise_diag"),
                    ("noise_s", "noise_s_diag"), ("y", "y")]:
        np.testing.assert_allclose(g[key], want[wk], rtol=1e-12)
    np.testing.assert_allclose(g["Z"], want["Z"][:, 0], rtol=1e-12)
    with pytest.raises(ag.DimensionMismatch):  # out_bar must be shaped like Z
        ag.posterior_rand_grad(p(ag.RowVecs(Xs), s2s), Z[:, 0], np.ones((M, 2)))
    with pytest.raises(ag.DimensionMismatch):
        ag.posterior_rand_grad(p(ag.RowVecs(Xs), s2s), Z[:-1, 0], Ob[:-1, 0])
    with pytest.raises(ag.AGPError):  # a FiniteGP over the prior is rand_grad's
        ag.posterior_rand_grad(ag.GP(ag.Matern52Kernel())(ag.RowVecs(X), s2), np.ones((N, 1)), np.ones((N, 1)))


def test_python_mirror_composite(fake_ag):
    """every kernel parameter's cotangent against central differences of the samples over refits"""
    ag, lib = fake_ag
    D, N, M, S = 1, 24, 8, 3
    X, y, Xs, _ = problem(N, M, D, 1, seed=2)
    Z, Ob = normals(M, S, 2)
    k = 0.8 * ag.with_lengthscale(ag.SqExponentialKernel(), 2.0) + 0.5 * ag.RationalQuadraticKernel(alpha=1.3)
    p = ag.posterior(ag.GP(k)(X[:, 0], 0.1), y)
    out, g = ag.posterior_rand_grad(p(Xs[:, 0], 0.05), Z, Ob)
    assert len(g["kernel"]) == len(ag.kernel_params(k))
    h = 1e-6
    vals = ag.kernel_params(k)

    def F(vv):
        kc = cr.from_struct(ag.api._kernel_struct(ag.with_kernel_params(k, vv), np.float64, [], D=D), D, np.float64)
        return float(np.sum(Ob * prr.post_rand_grad(kc, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, y, Xs, ref.MeanSpec(),
                                                    ref.NoiseSpec(0, 0.05), Z, Ob)["out"]))
    for i in range(len(vals)):
        vp, vm = list(vals), list(vals)
        vp[i], vm[i] = vals[i] + h, vals[i] - h
        fd = (F(vp) - F(vm)) / (2 * h)
        assert abs(g["kernel"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, g["kernel"][i], fd)


# ---- the C ABI and the Julia rule (the shim cannot be executed here: its structure is held to agp.h) --------------------
def test_cabi_prototype_matches_the_header(ag):
    restype, args = ag._cabi.SIGNATURES["agp_post_rand_grad"]
    assert len(args) == _header_arity("agp_post_rand_grad") == 18


POST_RAND_HEAD = ("function CRC.rrule(config::CRC.RuleConfig{>:CRC.HasReverseMode}, ::typeof(Random.rand), "
                  "rng::Random.AbstractRNG,\n                   fx::DevPostFiniteGP{T}, S::Int) where {T}")
PRIOR_RAND_HEAD = ("function CRC.rrule(config::CRC.RuleConfig{>:CRC.HasReverseMode}, ::typeof(Random.rand), "
                   "rng::Random.AbstractRNG,\n                   fx::DevFiniteGP{T}, S::Int) where {T}")
PULLBACK_HEAD = "function post_rand_rrule(rng, fx::DevPostFiniteGP{T}, S::Int, zero_mean::Bool) where {T}"


def test_julia_ccall_arity():
    """the argument-type tuple of the shim's ccall has one entry per parameter of the C prototype, and as many values"""
    src = _julia()
    head = "ccall((:agp_post_rand_grad, libagp), Int32,"
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
    assert commas + 1 == _header_arity("agp_post_rand_grad"), src[i:j + 1]
    rest = src[j + 1:src.index("))", j)]
    assert rest.count(",") - 1 == _header_arity("agp_post_rand_grad") - 1, rest


def test_julia_rule_follows_the_prior_rule():
    """the prior rule is found by the first occurrence of its head; the posterior rule comes after it"""
    src = _julia()
    assert src.count(PRIOR_RAND_HEAD) == 1 and src.count(POST_RAND_HEAD) == 1
    assert src.index(PRIOR_RAND_HEAD) < src.index(POST_RAND_HEAD)
    assert src.index("function CRC.rrule(config::CRC.RuleConfig{>:CRC.HasReverseMode}, ::typeof(Random.rand)") == \
        src.index(PRIOR_RAND_HEAD)


def test_julia_rule_forward_is_the_primal():
    """the primal method and the rule draw Z and sample through the same function"""
    src = _julia()
    assert ("Random.rand(rng::Random.AbstractRNG, fx::DevPostFiniteGP{T}, S::Int) where {T} = "
            "post_rand_primal(rng, fx, S, false)[1]") in src
    body = _rule(src, PULLBACK_HEAD)
    assert "post_rand_primal(rng, fx, S, zero_mean)" in body
    assert body.count("ccall((:agp_post_rand_grad, libagp)") == 1
    assert "Δ isa CRC.AbstractZero && return" in body
    assert body.index("AbstractZero") < body.index("convert(Matrix{T}, Δ)")
    for helper in ("kernel_tangent(", "composite_grads(", "mean_tangent(", "noise_tangent(", "x_tangent(", "as_storage("):
        assert helper in body, helper
    assert "C=(noise=g[4], noise_diag=nd)" in body and "δ=ȳ" in body
    assert "return CRC.NoTangent(), CRC.NoTangent(), f̄x, CRC.NoTangent()" in body


def test_julia_rule_splits_a_custom_mean():
    """a CustomMean prior goes through AD of the closure's values at x* plus a zero-test-mean device sample"""
    src = _julia()
    rule = _rule(src, POST_RAND_HEAD)
    assert ("fx.f.prior.mean isa AbstractGPs.CustomMean && return CRC.rrule_via_ad(config, mean_split_post_rand, rng, fx, S)"
            in rule)
    split = src[src.index("mean_split_post_rand(rng, fx::DevPostFiniteGP{T}, S::Int) where {T} ="):]
    split = split[:split.index("\n\n")]
    assert "AbstractGPs.mean_vector(fx.f.prior.mean, fx.x)" in split and "zero_mean_post_rand(rng, fx, S)" in split
    assert "mean_spec(AbstractGPs.ZeroMean(), fx.x, T)" in _rule(src, "function post_rand_primal(")
    assert ("CRC.rrule(::typeof(zero_mean_post_rand), rng::Random.AbstractRNG, fx::DevPostFiniteGP, S::Int) =\n"
            "    post_rand_rrule(rng, fx, S, true)") in src


def test_julia_tangents_name_only_primal_fields():
    found = _tangent_fields(_rule(_julia(), PULLBACK_HEAD))
    assert len(found) == 4
    for primal, names in found:
        assert primal in PRIMAL_FIELDS, primal
        assert names and set(names) <= PRIMAL_FIELDS[primal], (primal, names)
