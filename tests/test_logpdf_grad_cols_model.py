"""The gradient of sum_s w_s logpdf(fx, Y[:, s]) for a matrix Y (agp_post_logpdf_grad_cols) without a GPU: the NumPy model
tests/logpdf_grad_cols_ref.py pinned to torch fp64 autograd through torch.linalg.cholesky of an independent restatement
of logpdf, with every hyper-parameter, the noise, the mean, the inputs and Y as leaves; Ybar by central differences; the
single-column models at w = e_s; the Python mirror's argument passing through a stand-in library; ptxas on the new solve.cu
helpers; and the structure of the Julia rule."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import composite_ref as cr
import fake_libagp
import grad_x_ref as gx
import logpdf_grad_cols_ref as lc
from oracle import agp_ref as ref
from test_api_composite_fake import CompositeFakeLib
from test_grad_x_model import mauna_loa_shape
from test_rand_grad_model import _leaf, _torch_factor, single

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "abstractgps.jl_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]
RTOL = 1e-10


def torch_pullback(k, mean, noise, X, Y, w):
    """autograd of sum_s w_s logpdf(fx, Y[:, s]): (descriptor-order kernel gradient, noise, mean, x, Y)"""
    torch = pytest.importorskip("torch")
    kc = gx.as_composite(k)
    n = X.shape[0]
    Xt, Yt = _leaf(torch, X), _leaf(torch, Y)
    leaves = []
    K = torch.zeros((n, n), dtype=torch.float64)
    for v, fs in zip(kc.variance, kc.factors):
        vt = _leaf(torch, v)
        leaves.append(vt)
        P = vt * torch.ones((n, n), dtype=torch.float64)
        for F in fs:
            P = P * _torch_factor(torch, F, Xt, leaves)
        K = K + P
    s2 = _leaf(torch, noise.s if noise.kind == 0 else noise.v)
    Cm = K + torch.diag(s2 * torch.ones(n, dtype=torch.float64))
    mt = _leaf(torch, mean.c if mean.kind == 1 else (mean.v if mean.kind == 2 else 0.0))
    m = mt * torch.ones(n, dtype=torch.float64)
    L = torch.linalg.cholesky(Cm)
    Zq = torch.linalg.solve_triangular(L, Yt - m[:, None], upper=False)
    lp = -0.5 * (n * math.log(2 * math.pi) + 2.0 * torch.log(torch.diagonal(L)).sum() + (Zq * Zq).sum(0))
    (lp * torch.as_tensor(np.asarray(w, dtype=np.float64))).sum().backward()
    kg = np.concatenate([np.atleast_1d(t.grad.numpy()) for t in leaves])
    return kg, s2.grad.numpy(), mt.grad.numpy(), Xt.grad.numpy(), Yt.grad.numpy()


def problem(N, D, S, seed=0):
    rng = np.random.default_rng(seed + 13 * N + 5 * D + S)
    return rng.uniform(-2, 2, (N, D)), rng.standard_normal((N, S))


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


def _check(k, mean, noise, X, Y, w):
    got = lc.logpdf_grad_cols(k, mean, noise, X, Y, w)
    kg, ng, mg, xg, yg = torch_pullback(k, mean, noise, X, Y, w)
    if isinstance(k, cr.Composite):
        close(got["grad"][5:], kg)
    else:  # descriptor order of one factor: variance, Scale s | ARD v, Linear c
        g = got["grad"]
        want = [g[0]] + ([g[1]] if k.transform == cr.T_SCALE else []) + (list(g[5:]) if k.transform == cr.T_ARD else [])
        want += [g[2]] if k.family == cr.LINEAR else []
        close(np.array(want), kg)
        if k.transform != cr.T_SCALE:
            assert g[1] == 0.0
        if k.transform != cr.T_ARD:
            assert np.all(g[5:] == 0.0)
    close(got["noise_diag"] if noise.kind == 1 else got["grad"][3], ng)
    close(got["mean_diag"] if mean.kind == 2 else got["grad"][4], mg)
    close(got["x"], xg)
    close(got["Y"], yg)


@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_model_matches_torch_autograd(family, transform):
    D = 3
    k = single(family, transform, D, np.random.default_rng(family + 3 * transform))
    for S in (1, 3, 130):
        for wkind in ("ones", "mixed"):
            for noise_kind in (0, 1):
                for mean_kind in (0, 1, 2):
                    N = 30 + 2 * mean_kind + noise_kind
                    X, Y = problem(N, D, S, seed=family + mean_kind)
                    rng = np.random.default_rng(mean_kind + 3 * noise_kind)
                    mean = [ref.MeanSpec(), ref.MeanSpec(1, 0.3), ref.MeanSpec(2, v=rng.standard_normal(N))][mean_kind]
                    noise = ref.NoiseSpec(0, 0.1) if noise_kind == 0 else ref.NoiseSpec(1, v=rng.uniform(0.05, 0.2, N))
                    _check(k, mean, noise, X, Y, weights(S, wkind))


@pytest.mark.parametrize("D", [1, 3])
def test_model_matches_torch_autograd_mauna_loa(D):
    X, Y = problem(32, D, 3, seed=6)
    rng = np.random.default_rng(D)
    _check(mauna_loa_shape(D, rng), ref.MeanSpec(2, v=rng.standard_normal(32)), ref.NoiseSpec(1, v=rng.uniform(0.05, 0.2, 32)),
           X, Y, weights(3, "mixed"))


def test_ybar_matches_central_differences():
    """Ybar against central differences of sum_s w_s logpdf through the oracle's own logpdf"""
    k = single(cr.MATERN32, cr.T_ARD, 2, np.random.default_rng(0))
    X, Y = problem(25, 2, 4, seed=9)
    mean, noise, w = ref.MeanSpec(1, 0.2), ref.NoiseSpec(0, 0.1), weights(4, "mixed")
    got = lc.logpdf_grad_cols(k, mean, noise, X, Y, w)
    f = lambda YY: float(np.dot(w, ref.logpdf(k, mean, noise, X, YY)))  # noqa: E731
    h = 1e-6
    for i, s in [(0, 0), (7, 1), (24, 3), (12, 2)]:
        Yp, Ym = Y.copy(), Y.copy()
        Yp[i, s] += h
        Ym[i, s] -= h
        fd = (f(Yp) - f(Ym)) / (2 * h)
        assert abs(got["Y"][i, s] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, s, got["Y"][i, s], fd)


@pytest.mark.parametrize("kname", ["single", "mauna_loa"])
def test_unit_weight_is_the_single_column_model(kname):
    """w = e_s gives the single-column gradient of logpdf(fx, Y[:, s]): composite_ref.logpdf_grad for the parameters,
    grad_x_ref for the inputs, -alpha for y"""
    D = 2
    rng = np.random.default_rng(11)
    k = single(cr.SE, cr.T_SCALE, D, rng) if kname == "single" else mauna_loa_shape(D, rng)
    X, Y = problem(28, D, 5, seed=12)
    mean, noise = ref.MeanSpec(1, -0.4), ref.NoiseSpec(1, v=rng.uniform(0.05, 0.2, 28))
    kc = gx.as_composite(k)
    for s in (0, 2, 4):
        e = np.zeros(5)
        e[s] = 1.0
        got = lc.logpdf_grad_cols(k, mean, noise, X, Y, e)
        gd, gn = cr.logpdf_grad(kc, mean, noise, X, Y[:, s])
        if isinstance(k, cr.Composite):
            close(got["grad"], gd)
        else:
            close(got["grad"][0], gd[5])
            close(got["grad"][1], gd[6])
            close(got["grad"][3:5], gd[3:5])
        close(got["noise_diag"], gn)
        close(got["x"], gx.grad_x(k, mean, noise, X, Y[:, s]))
        close(lc.W_matrix(k, mean, noise, X, Y, e)[0], gx.W_matrix(k, mean, noise, X, Y[:, s]))
        assert np.all(got["Y"][:, [j for j in range(5) if j != s]] == 0.0)


# ---- the Python mirror through a stand-in library ---------------------------------------------------------------------
class ColsFakeLib(CompositeFakeLib):
    """answers agp_post_logpdf_grad_cols from the model and records the arguments"""

    def __init__(self):
        super().__init__()
        self.seen = []

    def agp_post_logpdf_grad_cols(self, p, ms, Y, S, lp_bar, g, nd, md, layout, xg, yb):
        post = self.posts[self._h(p)]
        dt = post["x"].dtype
        X = post["x"].astype(np.float64)
        n, D = X.shape
        if S < 1 or fake_libagp._addr(Y) is None or layout not in (0, 1):
            return self._fail(fake_libagp.INVALID, "invalid")
        mean = self._mean(ms, n, dt) if ms is not None else post["mean"]
        Ya = np.array(fake_libagp._arr(Y, (n, S), dt, "F"), dtype=np.float64)
        w = np.ones(S) if not lp_bar else np.array(np.ctypeslib.as_array(lp_bar, shape=(S,)))
        self.seen.append((S, None if not lp_bar else w.copy(), layout, fake_libagp._addr(nd) is not None,
                          fake_libagp._addr(md) is not None, fake_libagp._addr(xg) is not None, Ya.copy()))
        r = lc.logpdf_grad_cols(post["k"], mean, post["noise"], X, Ya, w)
        np.ctypeslib.as_array(g, shape=(len(r["grad"]),))[:] = r["grad"]
        for q, v, shape in [(nd, r["noise_diag"], (n,)), (md, r["mean_diag"], (n,)), (yb, r["Y"], (n, S))]:
            if fake_libagp._addr(q) is not None:
                fake_libagp._arr(q, shape, dt, "F")[...] = v
        if fake_libagp._addr(xg) is not None:  # in the input layout
            if layout == 0:
                fake_libagp._arr(xg, (n, D), dt)[...] = r["x"]
            else:
                fake_libagp._arr(xg, (n, D), dt, "F")[...] = r["x"]
        return 0


@pytest.fixture()
def fake_ag(ag, monkeypatch):
    eng = ag.api.Engine.__new__(ag.api.Engine)
    lib = ColsFakeLib()
    eng.L, eng.h, eng.device = lib, C.c_void_p(1), 0
    monkeypatch.setattr(ag.api, "_engine", eng)
    return ag, lib


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("container", ["row", "col", "vec"])
def test_python_mirror_passes_the_arguments(fake_ag, dtype, container):
    ag, lib = fake_ag
    D = 1 if container == "vec" else 2
    N, S = 20, 3
    X, Y = problem(N, D, S, seed=1)
    X, Y = X.astype(dtype), Y.astype(dtype)
    x = {"row": lambda: ag.RowVecs(X), "col": lambda: ag.ColVecs(X.T.copy()), "vec": lambda: X[:, 0].copy()}[container]()
    k = 1.3 * ag.with_lengthscale(ag.SqExponentialKernel(), 1 / 0.7)
    lp, g = ag.loglikelihood_grad(ag.GP(0.3, k)(x, 0.1), Y, inputs=True)
    S_, w, layout, has_nd, has_md, has_x, Ya = lib.seen[-1]
    assert (S_, w, layout, has_nd, has_md, has_x) == (S, None, 0, False, False, True)  # lp_bar=None -> NULL (all ones)
    np.testing.assert_array_equal(Ya, Y.astype(np.float64))
    X64 = X.astype(np.float64)
    want = lc.logpdf_grad_cols(ref.KernelSpec(cr.SE, 1.3, cr.T_SCALE, 0.7), ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X64,
                               Y.astype(np.float64))
    tol = 1e-10 if dtype == np.float64 else 1e-4
    assert lp.shape == (S,) and lp.dtype == dtype
    assert set(g) == {"variance", "scale", "noise", "mean_c", "Y", "x"}
    assert g["Y"].shape == (N, S) and g["Y"].dtype == dtype
    assert g["x"].shape == {"row": (N, D), "col": (D, N), "vec": (N,)}[container] and g["x"].dtype == dtype
    for key, i in [("variance", 0), ("scale", 1), ("noise", 3), ("mean_c", 4)]:
        np.testing.assert_allclose(g[key], want["grad"][i], rtol=tol)
    np.testing.assert_allclose(g["Y"], want["Y"], rtol=tol, atol=tol * np.abs(want["Y"]).max())
    xr = {"row": lambda: g["x"], "col": lambda: g["x"].T, "vec": lambda: g["x"][:, None]}[container]()
    np.testing.assert_allclose(xr, want["x"], rtol=tol, atol=tol * np.abs(want["x"]).max())
    np.testing.assert_allclose(lp, ref.logpdf(ref.KernelSpec(cr.SE, 1.3, cr.T_SCALE, 0.7), ref.MeanSpec(1, 0.3),
                                              ref.NoiseSpec(0, 0.1), X64, Y.astype(np.float64)), rtol=tol)


def test_python_mirror_weights_vector_y_custom_mean(fake_ag):
    """lp_bar reaches the call; a vector Y is one column; a CustomMean's values are passed again; per-point noise"""
    ag, lib = fake_ag
    N, D = 18, 2
    X, Y = problem(N, D, 1, seed=3)
    s2 = np.full(N, 0.1)
    fx = ag.GP(ag.CustomMean(lambda x: np.sin(x[0])), ag.Matern52Kernel())(ag.RowVecs(X), s2)
    lp, g = ag.loglikelihood_grad(fx, Y[:, 0], lp_bar=[-0.5])
    S_, w, layout, has_nd, has_md, has_x, _ = lib.seen[-1]
    assert S_ == 1 and list(w) == [-0.5] and has_nd and has_md and not has_x
    want = lc.logpdf_grad_cols(ref.KernelSpec(cr.MATERN52), ref.MeanSpec(2, v=np.sin(X[:, 0])), ref.NoiseSpec(1, v=s2), X,
                               Y, [-0.5])
    assert lp.shape == (1,) and g["Y"].shape == (N,) and g["noise"].shape == (N,) and "x" not in g
    np.testing.assert_allclose(g["mean_v"], want["mean_diag"], rtol=1e-12)
    np.testing.assert_allclose(g["noise"], want["noise_diag"], rtol=1e-12)
    np.testing.assert_allclose(g["Y"], want["Y"][:, 0], rtol=1e-12)
    with pytest.raises(ag.DimensionMismatch):
        ag.loglikelihood_grad(fx, Y[:, 0], lp_bar=[1.0, 2.0])
    with pytest.raises(ag.DimensionMismatch):
        ag.loglikelihood_grad(fx, Y[:-1])


def test_python_mirror_composite(fake_ag):
    ag, lib = fake_ag
    D, N, S = 1, 24, 3
    X, Y = problem(N, D, S, seed=2)
    k = 0.8 * ag.with_lengthscale(ag.SqExponentialKernel(), 2.0) + 0.5 * ag.RationalQuadraticKernel(alpha=1.3)
    w = np.array([1.0, -0.3, 2.0])
    lp, g = ag.loglikelihood_grad(ag.GP(k)(X[:, 0], 0.1), Y, lp_bar=w)
    assert len(g["kernel"]) == len(ag.kernel_params(k))
    h = 1e-6
    vals = ag.kernel_params(k)
    for i in range(len(vals)):  # every parameter's cotangent against central differences of the oracle's logpdf
        vp, vm = list(vals), list(vals)
        vp[i], vm[i] = vals[i] + h, vals[i] - h
        fp = np.dot(w, cr.logpdf(oracle_of_fake(ag, ag.with_kernel_params(k, vp), D), ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, Y))
        fm = np.dot(w, cr.logpdf(oracle_of_fake(ag, ag.with_kernel_params(k, vm), D), ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, Y))
        fd = (fp - fm) / (2 * h)
        assert abs(g["kernel"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, g["kernel"][i], fd)


def oracle_of_fake(ag, k, D):
    keep = []
    return cr.from_struct(ag.api._kernel_struct(k, np.float64, keep, D=D), D, np.float64)


def test_logpdf_grad_is_unchanged(fake_ag):
    """logpdf_grad keeps its single-column call and never reaches the new symbol"""
    ag, lib = fake_ag
    X, Y = problem(15, 2, 3, seed=4)
    lib.agp_post_logpdf_grad = lambda *a: CompositeFakeLib.agp_post_logpdf_grad(lib, *a)
    ag.logpdf_grad(ag.GP(ag.SqExponentialKernel() + ag.WhiteKernel())(ag.RowVecs(X), 0.1), Y[:, 0])
    assert lib.seen == []


# ---- the build ---------------------------------------------------------------------------------------------------------
def test_new_helpers_do_not_spill():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                        "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "solve.cu"), "-o", os.devnull],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", r.stderr)
    found = 0
    for b in blocks:
        if "sub_mean_cols_kernel" in b.split("\n", 1)[0] or "scale_kernel" in b.split("\n", 1)[0]:
            found += 1
            assert re.search(r"0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", b), b
    assert found == 4, r.stderr


# ---- the Julia rule (the shim cannot be executed here: its structure is held to what agp.h and the model establish) ------
def _julia_matrix_rule():
    src = open(os.path.join(ROOT, "julia", "AGPBlackwell.jl")).read()
    a = src.index("function CRC.rrule(::typeof(logpdf), fx::DevFiniteGP{T}, Y::AbstractMatrix{<:Real}) where {T}")
    return src, src[a:src.index("\nend\n", a)]


def test_julia_matrix_rule_is_behind_claimed():
    src, rule = _julia_matrix_rule()
    first = rule.split("\n")[1].strip()
    assert first.startswith("claimed(fx.f) || return nothing"), first
    # the forward pass keeps the handle, the pullback makes one call with lp_bar = the cotangent
    assert "lp, post = fit(fx, Y)" in rule
    assert rule.count("ccall((:agp_post_logpdf_grad_cols, libagp)") == 1
    assert "w = convert(Vector{Float64}, Δ)" in rule
    assert "post.data.C.h, ms, Ym, S, w, g, nd, C_NULL, layout, xg, Ȳ" in rule
    assert "return CRC.NoTangent(), f̄x, Ȳ" in rule
    # single kernels and trees are mapped back by the existing helpers
    for helper in ("kernel_tangent(", "composite_grads(", "ctangent(", "mean_tangent(", "noise_tangent(", "x_tangent("):
        assert helper in rule, helper
    # the vector rule is still there, unchanged in its signature
    assert "function CRC.rrule(::typeof(logpdf), fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}" in src
