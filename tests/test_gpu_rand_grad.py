"""The pullback of rand(fx, S) on the device (agp_rand_grad), in fp64 and fp32, against the CPU model tests/rand_grad_ref.py:
the five single-kernel families under every transform in the row, column and vector containers, per-point noise and a
vector mean, composites and the Mauna Loa kernel on the CO2 data, the int8-slice sizes, central differences of agp_rand
itself, the reference's own rand-gradient test, device memory, determinism, launch counts and the error codes.
Tolerances: rtol 1e-7 (fp64) / 2e-2 (fp32, against the model on the fp32-rounded inputs), atol the same times max|g|;
cond(C) <= 1e5.

fp32 problems are pulled back in fp64 on the problem converted to fp64 (agp.h).  The same pullback formed in fp32
arithmetic (numpy float32 throughout: Cholesky, L' Obar, Zbar Z', V = L^-1, V'QV), measured once on the CPU model at
N = 333, D = 3, S = 4, misses the fp64 result by 2.3e-4 of max|W| at cond(C) = 1.3e5 (SE, noise 1e-3), and the
contractions by 1.6e-4 (kernel), 3.9e-4 (noise) and 5.4e-5 (x); at cond(C) = 3e4 to 6e4 by 1e-5 to 4e-4."""
import ctypes as C

import numpy as np
import pytest

import composite_ref as cr
import rand_grad_ref as rg
from oracle import agp_ref as ref
from test_gpu_composite import KERNELS, _co2, _mauna_loa_kernel, oracle_of

pytestmark = pytest.mark.gpu
RT = {np.float64: 1e-7, np.float32: 2e-2}
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]


def data(N, D, S, dtype, seed=0):
    rng = np.random.default_rng(seed + 7 * N + D + 3 * S)
    X = rng.uniform(-2, 2, (N, D)).astype(dtype)
    return X, rng.standard_normal((N, S)).astype(dtype), rng.standard_normal((N, S)).astype(dtype)


def kernel(ag, family, transform, D):
    base = {cr.SE: ag.SqExponentialKernel, cr.MATERN12: ag.Matern12Kernel, cr.MATERN32: ag.Matern32Kernel,
            cr.MATERN52: ag.Matern52Kernel, cr.LINEAR: lambda: ag.LinearKernel(c=0.4)}[family]()
    ls = 1.5 * np.sqrt(D)
    ard = np.random.default_rng(D).uniform(0.5, 1.5, D) / ls
    if transform == cr.T_SCALE:
        base = ag.with_lengthscale(base, ls)
    elif transform == cr.T_ARD:
        base = base.compose(ag.ARDTransform(ard))
    spec = ref.KernelSpec(family, 1.3, transform, scale=1 / ls, ard=ard if transform == cr.T_ARD else None,
                          linear_c=0.4 if family == cr.LINEAR else 0.0)
    return 1.3 * base, spec


def close(got, want, rt):
    want = np.asarray(want, dtype=np.float64)
    got = np.asarray(got, dtype=np.float64)
    assert np.all(np.isfinite(got))
    np.testing.assert_allclose(got, want, rtol=rt, atol=rt * max(np.abs(want).max(), 1e-300))


def check_single(g, want, spec, rt):
    close(g["variance"], want["grad"][0], rt)
    if spec.transform == cr.T_SCALE:
        close(g["scale"], want["grad"][1], rt)
    elif spec.transform == cr.T_ARD:
        close(g["ard"], want["grad"][5:], rt)
    if spec.family == cr.LINEAR:
        close(g["linear_c"], want["grad"][2], rt)


def container(ag, X, kind):
    return {"row": lambda: ag.RowVecs(X), "col": lambda: ag.ColVecs(X.T.copy()), "vec": lambda: X[:, 0].copy()}[kind]()


def x_rows(xg, kind):
    return {"row": lambda: xg, "col": lambda: xg.T, "vec": lambda: xg[:, None]}[kind]()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_rand_grad_matches_model(ag, family, transform, dtype):
    rt = RT[dtype]
    for N, D, S, kind in [(10, 1, 1, "vec"), (63, 3, 3, "row"), (333, 1, 130, "col"), (333, 40, 4, "row"),
                          (1300, 3, 2, "col"), (1300, 40, 1, "row")]:
        k, spec = kernel(ag, family, transform, D)
        X, Z, Ob = data(N, D, S, dtype)
        out, g = ag.rand_grad(ag.GP(0.3, k)(container(ag, X, kind), 0.1), Z, Ob, inputs=True)
        X64, Z64, O64 = X.astype(np.float64), Z.astype(np.float64), Ob.astype(np.float64)
        want = rg.rand_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X64, Z64, O64)
        assert g["x"].dtype == dtype and g["Z"].dtype == dtype
        check_single(g, want, spec, rt)
        close(g["noise"], want["grad"][3], rt)
        close(g["mean_c"], want["grad"][4], rt)
        close(g["Z"], want["Z"], rt)
        close(x_rows(g["x"], kind), want["x"], rt)
        close(out, rg.rand(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X64, Z64), 10 * rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_per_point_noise_and_vector_mean(ag, dtype):
    N, D, S = 500, 2, 3
    k, spec = kernel(ag, cr.MATERN32, cr.T_ARD, D)
    X, Z, Ob = data(N, D, S, dtype, seed=1)
    s2 = np.random.default_rng(2).uniform(0.05, 0.2, N)
    out, g = ag.rand_grad(ag.GP(ag.CustomMean(lambda x: np.sin(x[0])), k)(ag.RowVecs(X), s2), Z, Ob, inputs=True)
    X64 = X.astype(np.float64)
    mv = np.sin(X64[:, 0].astype(dtype).astype(np.float64))
    want = rg.rand_grad(spec, ref.MeanSpec(2, v=mv), ref.NoiseSpec(1, v=s2.astype(dtype).astype(np.float64)), X64,
                        Z.astype(np.float64), Ob.astype(np.float64))
    rt = RT[dtype]
    close(g["noise"], want["noise_diag"], rt)
    close(g["mean_v"], want["mean_diag"], rt)
    close(g["x"], want["x"], rt)
    check_single(g, want, spec, rt)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname,D", [("stationary", 1), ("ard", 3), ("mixed", 3)])
def test_composite(ag, dtype, kname, D):
    k = KERNELS[kname](ag, D)
    ko = oracle_of(ag, k, D)
    X, Z, Ob = data(333, D, 3, dtype, seed=2)
    X[100] = X[7]  # coincident points (White, and the zero-difference convention)
    out, g = ag.rand_grad(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), Z, Ob, inputs=True)
    want = rg.rand_grad(ko, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X.astype(np.float64), Z.astype(np.float64),
                        Ob.astype(np.float64))
    rt = RT[dtype]
    wk = ag.api._Flat(k, D).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(w, dtype=np.float64)).max() for w in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(np.asarray(a, dtype=np.float64), b, rtol=rt, atol=rt * scale)
    close(g["noise"], want["grad"][3], rt)
    close(g["mean_c"], want["grad"][4], rt)
    close(g["x"], want["x"], rt)
    close(g["Z"], want["Z"], rt)


def test_mauna_loa(ag):
    x, y = _co2()
    xtr = x[:400]
    th0 = np.array([4.0, 4.0, 0.0, 1.0, 4.0, 0.0, 0.0, -1.0, -2.0, -2.0, -2.0])
    k = _mauna_loa_kernel(ag, th0)
    ko = oracle_of(ag, k, 1)
    rng = np.random.default_rng(3)
    Z, Ob = rng.standard_normal((400, 2)), rng.standard_normal((400, 2))
    out, g = ag.rand_grad(ag.GP(k)(xtr, 0.05), Z, Ob, inputs=True)
    want = rg.rand_grad(ko, ref.MeanSpec(), ref.NoiseSpec(0, 0.05), xtr[:, None], Z, Ob)
    wk = ag.api._Flat(k, 1).params_grad(want["grad"])
    scale = max(np.abs(np.asarray(w, dtype=np.float64)).max() for w in wk)
    for a, b in zip(g["kernel"], wk):
        np.testing.assert_allclose(a, b, rtol=1e-7, atol=1e-7 * scale)
    close(g["x"], want["x"][:, 0], 1e-7)
    close(g["noise"], want["grad"][3], 1e-7)


def _launches(ag, f):
    eng = ag.engine()
    c0 = eng.launch_count()
    r = f()
    return eng.launch_count() - c0, r


@pytest.mark.parametrize("dtype,N", [(np.float64, 8320), (np.float32, 4224)])
def test_int8_slice_sizes(ag, dtype, N):
    """fp64 N = 8320: the factor and V = L^-1 run on the int8-slice kernels; the fp32 problem's fp64 route at N = 4224:
    V = L^-1 does (the factor of an fp64 problem of that size stays on DMMA).  The branch is asserted from the launch
    counter: the automatic policy against tensor mode 0 on the same problem, results against the model."""
    eng = ag.engine()
    D, S = 2, 2
    k, spec = kernel(ag, cr.SE, cr.T_ARD, D)
    X, Z, Ob = data(N, D, S, dtype, seed=4)
    fx = ag.GP(0.3, k)(ag.RowVecs(X), 0.1)
    n_auto, (_, g) = _launches(ag, lambda: ag.rand_grad(fx, Z, Ob, inputs=True))
    cfg = eng.get_config()
    try:
        eng.set_config(fp64_mode=0)
        n_dmma, (_, g0) = _launches(ag, lambda: ag.rand_grad(fx, Z, Ob, inputs=True))
    finally:
        eng.set_config(fp64_mode=cfg.fp64_mode)
    assert n_auto != n_dmma, (n_auto, n_dmma)
    want = rg.rand_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.1), X.astype(np.float64), Z.astype(np.float64),
                        Ob.astype(np.float64))
    rt = RT[dtype]
    for gg in (g, g0):
        check_single(gg, want, spec, rt)
        close(gg["x"], want["x"], rt)
        close(gg["noise"], want["grad"][3], rt)


def test_central_differences_of_agp_rand(ag):
    """d/d variance, d/d scale, d/d noise and d/d x of sum(Obar o rand) against central differences of agp_rand itself"""
    N, D, S = 200, 2, 3
    X, Z, Ob = data(N, D, S, np.float64, seed=5)

    def f(v, ls, s2, XX):
        k = v * ag.with_lengthscale(ag.Matern52Kernel(), ls)
        return float(np.sum(Ob * ag.rand_from_normals(ag.GP(0.3, k)(ag.RowVecs(XX), s2), Z)))
    v, ls, s2 = 1.3, 1.7, 0.1
    _, g = ag.rand_grad(ag.GP(0.3, v * ag.with_lengthscale(ag.Matern52Kernel(), ls))(ag.RowVecs(X), s2), Z, Ob, inputs=True)
    h = 1e-6
    fd_v = (f(v + h, ls, s2, X) - f(v - h, ls, s2, X)) / (2 * h)
    s = 1 / ls
    fd_s = (f(v, 1 / (s + h), s2, X) - f(v, 1 / (s - h), s2, X)) / (2 * h)
    fd_n = (f(v, ls, s2 + h, X) - f(v, ls, s2 - h, X)) / (2 * h)
    Xp, Xm = X.copy(), X.copy()
    Xp[17, 1] += h
    Xm[17, 1] -= h
    fd_x = (f(v, ls, s2, Xp) - f(v, ls, s2, Xm)) / (2 * h)
    for a, b in [(g["variance"], fd_v), (g["scale"], fd_s), (g["noise"], fd_n), (g["x"][17, 1], fd_x)]:
        assert abs(a - b) <= 1e-6 * max(1.0, abs(b)), (a, b)


@pytest.mark.parametrize("S", [1, 3])
def test_reference_rand_gradient_replay(ag, S):
    """test/finite_gp_projection.jl:105-127: GP(sin, SE)(x, 1e-12), x = range(-3, 3, 10), the gradient with respect to x of
    <Obar, rand> at 1e-9, against torch fp64 autograd; the CustomMean sin is chained host-side through out["mean_v"]"""
    torch = pytest.importorskip("torch")
    N = 10
    x = np.linspace(-3.0, 3.0, N)
    rng = np.random.default_rng(123456)
    Z, Ob = rng.standard_normal((N, S)), rng.standard_normal((N, S))
    out, g = ag.rand_grad(ag.GP(ag.CustomMean(np.sin), ag.SqExponentialKernel())(x, 1e-12), Z, Ob, inputs=True)
    gx = g["x"] + np.cos(x) * g["mean_v"]
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    d2 = (xt[:, None] - xt[None, :]) ** 2
    L = torch.linalg.cholesky(torch.exp(-0.5 * d2) + 1e-12 * torch.eye(N, dtype=torch.float64))
    o = torch.sin(xt)[:, None] + L @ torch.as_tensor(Z)
    (o * torch.as_tensor(Ob)).sum().backward()
    np.testing.assert_allclose(out, o.detach().numpy(), rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(gx, xt.grad.numpy(), rtol=1e-9, atol=1e-9)


def _raw(ag, dtype, X, Z, Ob, nd=None, md=None, xg=None, zb=None, g=None, layout=0, S=None, k=None):
    cabi = ag._cabi
    keep = []
    ks = ag.api._kernel_struct(k or ag.with_lengthscale(ag.SqExponentialKernel(), 1.5), dtype, keep, D=X.shape[1])
    ms, ns = cabi.agp_mean(1, 0.3, None), cabi.agp_noise(0, 0.1, None)
    eng = ag.engine()
    gp = None if g is None else g.ctypes.data_as(C.POINTER(C.c_double))
    p = lambda a: a if isinstance(a, int) else cabi.ptr(a)  # noqa: E731
    return eng.L.agp_rand_grad(eng.h, cabi.dtype_code(dtype), C.byref(ks), C.byref(ms), C.byref(ns), layout, p(X),
                               X.shape[0], X.shape[1], p(Z), (Ob if Z is None else Z).shape[1] if S is None else S,
                               p(Ob), gp, p(nd), p(md), p(xg), p(zb))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_determinism_outputs_and_layouts(ag, dtype):
    """two calls give the same bits in every per-point output; NULL outputs are skipped; the feature-major layout is the
    transpose of the point-major one"""
    N, D, S = 700, 3, 4
    X, Z, Ob = data(N, D, S, dtype, seed=6)
    Xc, Zf, Of = np.ascontiguousarray(X), np.asfortranarray(Z), np.asfortranarray(Ob)
    outs = []
    for _ in range(2):
        g, nd, md = np.zeros(5 + D), np.empty(N, dtype=dtype), np.empty(N, dtype=dtype)
        xg, zb = np.empty((N, D), dtype=dtype), np.empty((N, S), dtype=dtype, order="F")
        assert _raw(ag, dtype, Xc, Zf, Of, nd, md, xg, zb, g) == 0
        outs.append((g, nd, md, xg, zb))
    for a, b in zip(outs[0][1:], outs[1][1:]):
        assert a.tobytes() == b.tobytes()
    assert outs[0][0][4] == outs[1][0][4]  # sum of mean_diag in index order
    np.testing.assert_allclose(outs[0][0], outs[1][0], rtol=1e-12, atol=1e-12 * np.abs(outs[0][0]).max())
    zb = np.empty((N, S), dtype=dtype, order="F")
    assert _raw(ag, dtype, Xc, Zf, Of, zb=zb) == 0  # only z_bar: V, Q and the reductions are skipped
    assert zb.tobytes() == outs[0][4].tobytes()
    xf = np.empty((N, D), dtype=dtype, order="F")
    assert _raw(ag, dtype, np.asfortranarray(X), Zf, Of, xg=xf, layout=1) == 0
    assert xf.tobytes(order="F") == np.asfortranarray(outs[0][3]).tobytes(order="F")


def test_device_memory(ag):
    torch = pytest.importorskip("torch")
    cabi = ag._cabi
    eng = ag.engine()
    N, D, S = 500, 4, 3
    X, Z, Ob = data(N, D, S, np.float64, seed=7)
    Xc, Zf, Of = np.ascontiguousarray(X), np.asfortranarray(Z), np.asfortranarray(Ob)
    g0, nd0, md0, xg0, zb0 = np.zeros(5 + D), np.empty(N), np.empty(N), np.empty((N, D)), np.empty((N, S), order="F")
    assert _raw(ag, np.float64, Xc, Zf, Of, nd0, md0, xg0, zb0, g0) == 0
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a.ravel(order="K"))).cuda()  # noqa: E731
    Xd, Zd, Od = dev(Xc), torch.from_numpy(Zf.ravel(order="F").copy()).cuda(), torch.from_numpy(Of.ravel(order="F").copy()).cuda()
    nd, md, xg, zb = (torch.empty(n, dtype=torch.float64, device="cuda") for n in (N, N, N * D, N * S))
    g = np.zeros(5 + D)
    torch.cuda.synchronize()
    eng.set_memspace(cabi.AGP_MEM_DEVICE)
    try:
        rc = _raw(ag, np.float64, _DevArr(Xd, N, D), _DevArr(Zd, N, S), _DevArr(Od, N, S), nd.data_ptr(), md.data_ptr(),
                  xg.data_ptr(), zb.data_ptr(), g)
    finally:
        eng.set_memspace(cabi.AGP_MEM_HOST)
    assert rc == 0
    assert nd.cpu().numpy().tobytes() == nd0.tobytes() and md.cpu().numpy().tobytes() == md0.tobytes()
    assert xg.cpu().numpy().tobytes() == xg0.tobytes() and zb.cpu().numpy().tobytes() == zb0.tobytes(order="F")
    np.testing.assert_allclose(g, g0, rtol=1e-12, atol=1e-12 * np.abs(g0).max())


class _DevArr(int):
    """a device address that also carries the shape _raw reads"""

    def __new__(cls, t, n, m):
        o = int.__new__(cls, t.data_ptr())
        o.shape = (n, m)
        o._t = t
        return o


def test_agp_rand_launches_unchanged(ag):
    """agp_rand is the factor-only fit plus the TRMM and the mean: its launch count is the fit's + 2 (+1 without a mean)"""
    cabi = ag._cabi
    eng = ag.engine()
    N, D, S = 600, 2, 3
    X, Z, Ob = data(N, D, S, np.float64, seed=8)
    keep = []
    ks = ag.api._kernel_struct(ag.SqExponentialKernel(), np.float64, keep, D=D)
    ns = cabi.agp_noise(0, 0.1, None)
    Xc, Zf = np.ascontiguousarray(X), np.asfortranarray(Z)
    out = np.empty((N, S), order="F")
    for mean, extra in [(cabi.agp_mean(0, 0.0, None), 1), (cabi.agp_mean(1, 0.3, None), 2)]:
        n_fit, rc = _launches(ag, lambda: eng.L.agp_fit(eng.h, 1, C.byref(ks), C.byref(mean), C.byref(ns), 0, cabi.ptr(Xc), N, D,
                                                        None, 0, None, None, None))
        assert rc == 0
        n_rand, rc = _launches(ag, lambda: eng.L.agp_rand(eng.h, 1, C.byref(ks), C.byref(mean), C.byref(ns), 0, cabi.ptr(Xc), N,
                                                          D, cabi.ptr(Zf), S, cabi.ptr(out)))
        assert rc == 0
        assert n_rand == n_fit + extra, (n_rand, n_fit, extra)


def test_launches_against_the_logpdf_gradient(ag):
    """the pullback is the factor-only fit, the logpdf gradient's substitution and reductions, and six launches of its own
    (the row sum, the export of L', L' Obar, Zbar Z', the mirror, Q V; V' W1 takes the place of the logpdf gradient's V'V)"""
    cabi = ag._cabi
    eng = ag.engine()
    N, D, S = 3000, 2, 3
    X, Z, Ob = data(N, D, S, np.float64, seed=9)
    Xc, Zf, Of = np.ascontiguousarray(X), np.asfortranarray(Z), np.asfortranarray(Ob)
    keep = []
    k = ag.with_lengthscale(ag.SqExponentialKernel(), 1.5)
    ks = ag.api._kernel_struct(k, np.float64, keep, D=D)
    ms, ns = cabi.agp_mean(1, 0.3, None), cabi.agp_noise(0, 0.1, None)
    n_fit, rc = _launches(ag, lambda: eng.L.agp_fit(eng.h, 1, C.byref(ks), C.byref(ms), C.byref(ns), 0, cabi.ptr(Xc), N, D,
                                                    None, 0, None, None, None))
    assert rc == 0
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), np.zeros(N))
    g, nd, xg = np.zeros(5 + D), np.empty(N), np.empty((N, D))
    n_lg, rc = _launches(ag, lambda: eng.L.agp_post_logpdf_grad_x(post.data.C.h, g.ctypes.data_as(C.POINTER(C.c_double)),
                                                                  cabi.ptr(nd), 0, cabi.ptr(xg)))
    assert rc == 0
    n_rg, rc = _launches(ag, lambda: _raw(ag, np.float64, Xc, Zf, Of, nd, None, xg, None, g, k=k))
    assert rc == 0
    assert n_rg == n_fit + n_lg + 6, (n_rg, n_fit, n_lg)


def test_errors(ag):
    cabi = ag._cabi
    eng = ag.engine()
    N, D, S = 50, 2, 2
    X, Z, Ob = data(N, D, S, np.float64, seed=10)
    Xc, Zf, Of = np.ascontiguousarray(X), np.asfortranarray(Z), np.asfortranarray(Ob)
    g = np.zeros(5 + D)
    assert _raw(ag, np.float64, Xc, Zf, Of, g=g, layout=2) == cabi.AGP_ERR_INVALID
    assert _raw(ag, np.float64, Xc, Zf, None, g=g) == cabi.AGP_ERR_INVALID
    assert _raw(ag, np.float64, Xc, None, Of, g=g) == cabi.AGP_ERR_INVALID
    assert _raw(ag, np.float64, Xc, Zf, Of, g=g, S=-1) == cabi.AGP_ERR_INVALID
    # a C that is not positive definite: K - 2 I fails at the first pivot (K_11 = 1)
    keep = []
    ks = ag.api._kernel_struct(ag.SqExponentialKernel(), np.float64, keep, D=D)
    ms, ns = cabi.agp_mean(0, 0.0, None), cabi.agp_noise(0, -2.0, None)
    rc = eng.L.agp_rand_grad(eng.h, 1, C.byref(ks), C.byref(ms), C.byref(ns), 0, cabi.ptr(Xc), N, D, cabi.ptr(Zf), S,
                             cabi.ptr(Of), g.ctypes.data_as(C.POINTER(C.c_double)), None, None, None, None)
    assert rc == cabi.AGP_ERR_NOT_POSDEF
    assert eng.L.agp_last_info(eng.h) > 0
    # the context still works
    assert _raw(ag, np.float64, Xc, Zf, Of, g=g) == 0
    # S = 0: every output is zero
    g0 = np.full(5 + D, 7.0)
    assert _raw(ag, np.float64, Xc, Zf, Of, g=g0, S=0) == 0
    assert np.all(g0 == 0.0)
