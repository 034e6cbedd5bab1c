"""The pullback of rand(fx, S) (agp_rand_grad) without a GPU: the NumPy model tests/rand_grad_ref.py pinned to torch fp64
autograd through torch.linalg.cholesky of an independent restatement of out = m + chol(K + Sigma_y) Z, with every
hyper-parameter, the noise, the mean, the inputs and the normals as leaves; the Python mirror's argument passing through a
stand-in library; and ptxas on rand_grad.cu."""
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
import rand_grad_ref as rg
from oracle import agp_ref as ref
from test_api_composite_fake import CompositeFakeLib
from test_grad_x_model import mauna_loa_shape

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "abstractgps.jl_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]
RTOL = 1e-10


# ---- an independent torch restatement of rand -------------------------------------------------------------------------
def _leaf(torch, v):
    return torch.tensor(np.asarray(v, dtype=np.float64), dtype=torch.float64, requires_grad=True)


def _torch_factor(torch, F, X, leaves):
    """kappa_f on X (N x D tensor) from the KernelFunctions definitions; every parameter of F is a new leaf appended to
    `leaves` in the agp_post_logpdf_grad order of the factor: Scale s | ARD v, then param, then Periodic r"""
    n, D = X.shape
    eye = torch.eye(n, dtype=torch.bool)
    if F.transform == cr.T_SCALE:
        t = _leaf(torch, F.scale)
        leaves.append(t)
        A = X * t
    elif F.transform == cr.T_ARD:
        t = _leaf(torch, F.ard)
        leaves.append(t)
        A = X * t
    else:
        A = X
    p = None
    if F.family in (cr.RQ, cr.LINEAR, cr.CONSTANT):
        p = _leaf(torch, F.param)
        leaves.append(p)
    if F.family == cr.CONSTANT:
        return p * torch.ones((n, n), dtype=torch.float64)
    if F.family == cr.LINEAR:
        return A @ A.T + p
    diff = A[:, None, :] - A[None, :, :]
    if F.family == cr.PERIODIC:
        r = _leaf(torch, np.ones(D) if F.r is None else F.r)
        leaves.append(r)
        s = torch.sin(math.pi * diff) / r
        return torch.exp(-0.5 * (s * s).sum(2))
    d2 = (diff * diff).sum(2)
    if F.family == cr.WHITE:
        return eye.to(torch.float64)
    if F.family == cr.SE:
        return torch.exp(-0.5 * d2)
    if F.family == cr.RQ:
        return (1.0 + d2 / (2.0 * p)) ** (-p)
    d = torch.sqrt(torch.where(eye, torch.ones_like(d2), d2))  # the points are distinct: only the diagonal is 0
    if F.family == cr.MATERN12:
        k = torch.exp(-d)
    elif F.family == cr.MATERN32:
        k = (1.0 + math.sqrt(3.0) * d) * torch.exp(-math.sqrt(3.0) * d)
    else:
        s5 = math.sqrt(5.0) * d
        k = (1.0 + s5 + s5 * s5 / 3.0) * torch.exp(-s5)
    return torch.where(eye, torch.ones_like(k), k)


def torch_pullback(k, mean, noise, X, Z, Obar):
    """autograd of sum(Obar o (m + L Z)): (descriptor-order kernel gradient, noise, mean, x, Z)"""
    torch = pytest.importorskip("torch")
    kc = gx.as_composite(k)
    n = X.shape[0]
    Xt, Zt = _leaf(torch, X), _leaf(torch, Z)
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
    out = m[:, None] + L @ Zt
    (out * torch.as_tensor(Obar)).sum().backward()
    kg = np.concatenate([np.atleast_1d(t.grad.numpy()) for t in leaves])
    return kg, s2.grad.numpy(), mt.grad.numpy(), Xt.grad.numpy(), Zt.grad.numpy()


def single(family, transform, D, rng):
    ard = rng.uniform(0.5, 1.5, D) if transform == cr.T_ARD else None
    return ref.KernelSpec(family, 1.3, transform, scale=0.7, ard=ard, linear_c=0.4 if family == cr.LINEAR else 0.0)


def problem(N, D, S, seed=0):
    rng = np.random.default_rng(seed + 13 * N + 5 * D + S)
    return rng.uniform(-2, 2, (N, D)), rng.standard_normal((N, S)), rng.standard_normal((N, S))


def _check(k, mean, noise, X, Z, Obar):
    got = rg.rand_grad(k, mean, noise, X, Z, Obar)
    kg, ng, mg, xg, zg = torch_pullback(k, mean, noise, X, Z, Obar)
    D = X.shape[1]

    def close(a, b):
        b = np.asarray(b, dtype=np.float64)
        np.testing.assert_allclose(a, b, rtol=RTOL, atol=RTOL * max(1.0, np.abs(b).max()))
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
    if mean.kind == 1:
        close(got["grad"][4], mg)
    elif mean.kind == 2:
        close(got["mean_diag"], mg)
    close(got["x"], xg)
    close(got["Z"], zg)
    # the forward pass the pullback belongs to is agp_rand's (the oracle)
    if isinstance(k, ref.KernelSpec):
        np.testing.assert_allclose(rg.rand(k, mean, noise, X, Z), ref.rand_from_Z(k, mean, noise, X, Z), rtol=1e-12,
                                   atol=1e-12)


@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_model_matches_torch_autograd(family, transform):
    D = 3
    k = single(family, transform, D, np.random.default_rng(family + 3 * transform))
    for i, (N, S, mean, noise_kind) in enumerate([(30, 3, ref.MeanSpec(1, 0.3), 0), (34, 1, ref.MeanSpec(), 1),
                                                   (36, 4, None, 0)]):
        X, Z, Obar = problem(N, D, S, seed=family + i)
        rng = np.random.default_rng(i)
        if mean is None:
            mean = ref.MeanSpec(2, v=rng.standard_normal(N))
        noise = ref.NoiseSpec(0, 0.1) if noise_kind == 0 else ref.NoiseSpec(1, v=rng.uniform(0.05, 0.2, N))
        _check(k, mean, noise, X, Z, Obar)


def test_model_matches_torch_autograd_many_columns():
    """S = 130: more normals than the border tile of the factorisation carries"""
    k = single(cr.MATERN52, cr.T_ARD, 2, np.random.default_rng(4))
    X, Z, Obar = problem(40, 2, 130, seed=3)
    _check(k, ref.MeanSpec(1, -0.2), ref.NoiseSpec(0, 0.05), X, Z, Obar)


@pytest.mark.parametrize("D", [1, 3])
def test_model_matches_torch_autograd_mauna_loa(D):
    X, Z, Obar = problem(32, D, 3, seed=6)
    rng = np.random.default_rng(D)
    _check(mauna_loa_shape(D, rng), ref.MeanSpec(2, v=rng.standard_normal(32)), ref.NoiseSpec(1, v=rng.uniform(0.05, 0.2, 32)),
           X, Z, Obar)


def test_model_matches_central_differences():
    """the whole chain once more against the oracle's own rand: d/d variance, d/d noise and d/d x of sum(Obar o out)"""
    k = single(cr.SE, cr.T_SCALE, 2, np.random.default_rng(0))
    X, Z, Obar = problem(25, 2, 3, seed=9)
    mean, noise = ref.MeanSpec(1, 0.2), ref.NoiseSpec(0, 0.1)
    got = rg.rand_grad(k, mean, noise, X, Z, Obar)
    f = lambda kk, nn, XX: float(np.sum(Obar * ref.rand_from_Z(kk, mean, nn, XX, Z)))  # noqa: E731
    h = 1e-6
    kp, km = ref.KernelSpec(**{**k.__dict__, "variance": k.variance + h}), ref.KernelSpec(**{**k.__dict__, "variance": k.variance - h})
    fd = (f(kp, noise, X) - f(km, noise, X)) / (2 * h)
    assert abs(got["grad"][0] - fd) <= 1e-6 * max(1.0, abs(fd))
    fd = (f(k, ref.NoiseSpec(0, 0.1 + h), X) - f(k, ref.NoiseSpec(0, 0.1 - h), X)) / (2 * h)
    assert abs(got["grad"][3] - fd) <= 1e-6 * max(1.0, abs(fd))
    Xp, Xm = X.copy(), X.copy()
    Xp[7, 1] += h
    Xm[7, 1] -= h
    fd = (f(k, noise, Xp) - f(k, noise, Xm)) / (2 * h)
    assert abs(got["x"][7, 1] - fd) <= 1e-6 * max(1.0, abs(fd))


# ---- the Python mirror through a stand-in library ---------------------------------------------------------------------
class RandGradFakeLib(CompositeFakeLib):
    """answers agp_rand / agp_rand_grad from the model and records the arguments"""

    def __init__(self):
        super().__init__()
        self.seen = []

    def _problem(self, code, ks, ms, ns, layout, X, n, D):
        dt = self._dt(code)
        return dt, self._kernel(ks, D, dt), self._mean(ms, n, dt), self._noise(ns, n, dt), self._points(layout, X, n, D, dt)

    def agp_rand(self, h, code, ks, ms, ns, layout, X, n, D, Z, S, out):
        dt, k, mean, noise, Xa = self._problem(code, ks, ms, ns, layout, X, n, D)
        fake_libagp._arr(out, (n, S), dt, "F")[...] = rg.rand(k, mean, noise, Xa, np.array(fake_libagp._arr(Z, (n, S), dt, "F")))
        return 0

    def agp_rand_grad(self, h, code, ks, ms, ns, layout, X, n, D, Z, S, Ob, g, nd, md, xg, zb):
        dt, k, mean, noise, Xa = self._problem(code, ks, ms, ns, layout, X, n, D)
        Za, Oa = np.array(fake_libagp._arr(Z, (n, S), dt, "F")), np.array(fake_libagp._arr(Ob, (n, S), dt, "F"))
        self.seen.append((layout, S, fake_libagp._addr(nd) is not None, fake_libagp._addr(md) is not None,
                          fake_libagp._addr(xg) is not None))
        r = rg.rand_grad(k, mean, noise, Xa, Za, Oa)
        np.ctypeslib.as_array(g, shape=(len(r["grad"]),))[:] = r["grad"]
        for p, v, shape in [(nd, r["noise_diag"], (n,)), (md, r["mean_diag"], (n,)), (zb, r["Z"], (n, S))]:
            if fake_libagp._addr(p) is not None:
                fake_libagp._arr(p, shape, dt, "F")[...] = v
        if fake_libagp._addr(xg) is not None:  # in the input layout
            if layout == 0:
                fake_libagp._arr(xg, (n, D), dt)[...] = r["x"]
            else:
                fake_libagp._arr(xg, (n, D), dt, "F")[...] = r["x"]
        return 0


@pytest.fixture()
def fake_ag(ag, monkeypatch):
    eng = ag.api.Engine.__new__(ag.api.Engine)
    lib = RandGradFakeLib()
    eng.L, eng.h, eng.device = lib, C.c_void_p(1), 0
    monkeypatch.setattr(ag.api, "_engine", eng)
    return ag, lib


def test_python_mirror_passes_the_arguments(fake_ag):
    ag, lib = fake_ag
    D, N, S = 2, 20, 3
    X, Z, Obar = problem(N, D, S, seed=1)
    k = 1.3 * ag.with_lengthscale(ag.SqExponentialKernel(), 1 / 0.7)
    fx = ag.GP(0.3, k)(ag.RowVecs(X), 0.1)
    out, g = ag.rand_grad(fx, Z, Obar, inputs=True)
    want = rg.rand_grad(ref.KernelSpec(cr.SE, 1.3, cr.T_SCALE, 0.7), ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X, Z, Obar)
    assert lib.seen[-1] == (0, S, False, False, True)
    np.testing.assert_allclose(g["variance"], want["grad"][0], rtol=1e-12)
    np.testing.assert_allclose(g["scale"], want["grad"][1], rtol=1e-12)
    np.testing.assert_allclose(g["noise"], want["grad"][3], rtol=1e-12)
    np.testing.assert_allclose(g["mean_c"], want["grad"][4], rtol=1e-12)
    np.testing.assert_allclose(g["Z"], want["Z"], rtol=1e-12)
    assert g["x"].shape == (N, D)
    np.testing.assert_allclose(g["x"], want["x"], rtol=1e-12, atol=1e-14)
    # a vector Z, ColVecs, per-point noise and a CustomMean
    s2 = np.full(N, 0.1)
    fx = ag.GP(ag.CustomMean(lambda x: np.sin(x[0])), k)(ag.ColVecs(X.T.copy()), s2)
    out, g = ag.rand_grad(fx, Z[:, 0], Obar[:, 0], inputs=True)
    assert lib.seen[-1] == (0, 1, True, True, True)
    want = rg.rand_grad(ref.KernelSpec(cr.SE, 1.3, cr.T_SCALE, 0.7), ref.MeanSpec(2, v=np.sin(X[:, 0])),
                        ref.NoiseSpec(1, v=s2), X, Z[:, :1], Obar[:, :1])
    assert g["Z"].shape == (N,) and g["x"].shape == (D, N) and g["noise"].shape == (N,)
    np.testing.assert_allclose(g["mean_v"], want["mean_diag"], rtol=1e-12)
    np.testing.assert_allclose(g["noise"], want["noise_diag"], rtol=1e-12)
    np.testing.assert_allclose(g["x"], want["x"].T, rtol=1e-12, atol=1e-14)


def test_python_mirror_composite(fake_ag):
    ag, lib = fake_ag
    D, N, S = 1, 24, 2
    X, Z, Obar = problem(N, D, S, seed=2)
    k = 0.8 * ag.with_lengthscale(ag.SqExponentialKernel(), 2.0) + 0.5 * ag.RationalQuadraticKernel(alpha=1.3)
    out, g = ag.rand_grad(ag.GP(k)(X[:, 0], 0.1), Z, Obar)
    assert len(g["kernel"]) == len(ag.kernel_params(k))
    h = 1e-6
    vals = ag.kernel_params(k)
    for i in range(len(vals)):  # every parameter's cotangent against central differences of the model's rand
        vp, vm = list(vals), list(vals)
        vp[i], vm[i] = vals[i] + h, vals[i] - h
        fp = np.sum(Obar * rg.rand(oracle_of_fake(ag, ag.with_kernel_params(k, vp), D), ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, Z))
        fm = np.sum(Obar * rg.rand(oracle_of_fake(ag, ag.with_kernel_params(k, vm), D), ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, Z))
        fd = (fp - fm) / (2 * h)
        assert abs(g["kernel"][i] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, g["kernel"][i], fd)


def oracle_of_fake(ag, k, D):
    keep = []
    return cr.from_struct(ag.api._kernel_struct(k, np.float64, keep, D=D), D, np.float64)


# ---- the build ---------------------------------------------------------------------------------------------------------
def test_rand_grad_kernels_do_not_spill():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                        "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "rand_grad.cu"), "-o", os.devnull],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame", r.stderr)
    assert spills and all(a == "0" and b == "0" for a, b in spills), r.stderr
    assert frames and all(f == "0" for f in frames), r.stderr


# ---- the Julia rule (the shim cannot be executed here: its structure is held to what agp.h and the model establish) ------
def _julia_rand_rule():
    src = open(os.path.join(ROOT, "julia", "AGPBlackwell.jl")).read()
    a = src.index("function CRC.rrule(config::CRC.RuleConfig{>:CRC.HasReverseMode}, ::typeof(Random.rand)")
    return src, src[a:src.index("\nend\n", a)]


def test_julia_rand_rule_differentiates_a_custom_mean():
    """agp_rand_grad treats a vector mean as a constant of x; the rule must not hand such a prior to it, or the closure's
    term cos(x) .* sum(Obar, dims=2) of the reference's rand-gradient test would be lost.  The rule sends a CustomMean prior
    through AD of `mean_split_rand`: the closure's values plus a sample of the zero-mean prior"""
    src, rule = _julia_rand_rule()
    assert "fx.f.mean isa AbstractGPs.CustomMean && return CRC.rrule_via_ad(config, mean_split_rand, rng, fx, S)" in rule
    assert rule.index("CustomMean") < rule.index("agp_rand_grad")
    split = src[src.index("mean_split_rand(rng, fx::DevFiniteGP{T}, S) where {T} ="):]
    split = split[:split.index("\n\n")]
    assert "AbstractGPs.mean_vector(fx.f.mean, fx.x)" in split and "GP(AbstractGPs.ZeroMean(), fx.f.kernel)" in split


def test_julia_rand_rule_accepts_a_zero_cotangent():
    _, rule = _julia_rand_rule()
    assert "Δ isa CRC.AbstractZero && return" in rule
    assert rule.index("AbstractZero") < rule.index("convert(Matrix{T}")
