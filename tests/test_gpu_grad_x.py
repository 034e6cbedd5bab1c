"""The gradient of logpdf with respect to the input points on the device (agp_post_logpdf_grad_x), in fp64 and fp32,
against the CPU model tests/grad_x_ref.py: the five single-kernel families under every transform, composites, the
int8-slice Cholesky sizes, determinism and agreement with agp_post_logpdf_grad, device memory, errors, the reference's
own input-gradient check and a deep-kernel-learning replay through a torch network.
Tolerances: rtol 1e-7 (fp64) / 2e-2 (fp32, against the model on the fp32-rounded inputs), atol the same times max|g|."""
import ctypes as C
import os

import numpy as np
import pytest

import composite_ref as cr
import grad_x_ref as gx
from oracle import agp_ref as ref
from test_gpu_composite import KERNELS, _co2, _mauna_loa_kernel, oracle_of

pytestmark = pytest.mark.gpu
RT = {np.float64: 1e-7, np.float32: 2e-2}
FAMILIES = [cr.SE, cr.MATERN12, cr.MATERN32, cr.MATERN52, cr.LINEAR]


def data(N, D, dtype, seed=0):
    rng = np.random.default_rng(seed + 7 * N + D)
    X = rng.uniform(-2, 2, (N, D)).astype(dtype)
    y = (np.sin(2 * X.astype(np.float64)).sum(1) + 0.1 * rng.normal(size=N)).astype(dtype)
    return X, y


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


def check(g, X64, ko, y, s2, c, dtype):
    want = gx.grad_x(ko, ref.MeanSpec(1, c), ref.NoiseSpec(0, s2), X64, y.astype(np.float64))
    rt = RT[dtype]
    np.testing.assert_allclose(g, want, rtol=rt, atol=rt * np.abs(want).max())
    assert np.all(np.isfinite(g))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform", [cr.T_NONE, cr.T_SCALE, cr.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_grad_x_matches_model(ag, family, transform, dtype):
    for N, D, container in [(1, 1, "vec"), (63, 3, "row"), (333, 1, "col"), (333, 40, "row"), (1300, 1, "col"),
                            (1300, 3, "row"), (1300, 40, "col")]:
        k, ko = kernel(ag, family, transform, D)
        X, y = data(N, D, dtype)
        x = {"row": lambda: ag.RowVecs(X), "col": lambda: ag.ColVecs(X.T.copy()), "vec": lambda: X[:, 0].copy()}[container]()
        s2 = 0.1
        lp, g = ag.logpdf_grad(ag.GP(0.3, k)(x, s2), y, inputs=True)
        gx_ = {"row": lambda: g["x"], "col": lambda: g["x"].T, "vec": lambda: g["x"][:, None]}[container]()
        assert g["x"].dtype == dtype
        check(gx_, X.astype(np.float64), ko, y, s2, 0.3, dtype)


@pytest.mark.parametrize("dtype,N", [(np.float64, 8320), (np.float32, 4224)])
def test_grad_x_on_int8_slice_cholesky(ag, dtype, N):
    D = 2
    k, ko = kernel(ag, cr.SE, cr.T_ARD, D)
    X, y = data(N, D, dtype)
    lp, g = ag.logpdf_grad(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y, inputs=True)
    check(g["x"], X.astype(np.float64), ko, y, 0.1, 0.3, dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname,D", [("stationary", 1), ("stationary", 3), ("ard", 3), ("mixed", 3)])
def test_composite_grad_x(ag, dtype, kname, D):
    k = KERNELS[kname](ag, D)
    ko = oracle_of(ag, k, D)
    X, y = data(333, D, dtype, seed=2)
    X[100] = X[7]  # coincident points (White, and the zero-difference convention)
    lp, g = ag.logpdf_grad(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y, inputs=True)
    check(g["x"], X.astype(np.float64), ko, y, 0.1, 0.3, dtype)


def test_mauna_loa_grad_x(ag):
    x, y = _co2()
    xtr, ytr = x[:400], y[:400]
    th0 = np.array([4.0, 4.0, 0.0, 1.0, 4.0, 0.0, 0.0, -1.0, -2.0, -2.0, -2.0])
    k = _mauna_loa_kernel(ag, th0)
    ko = oracle_of(ag, k, 1)
    lp, g = ag.logpdf_grad(ag.GP(k)(xtr, 0.05), ytr, inputs=True)
    want = gx.grad_x(ko, ref.MeanSpec(), ref.NoiseSpec(0, 0.05), xtr[:, None], ytr)[:, 0]
    np.testing.assert_allclose(g["x"], want, rtol=1e-7, atol=1e-7 * np.abs(want).max())


def _handle(ag, k, X, y, s2=0.1):
    return ag.posterior(ag.GP(k)(ag.RowVecs(X), s2), y)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kname", ["se_ard", "composite"])
def test_determinism_and_agreement_with_hyper_gradient(ag, dtype, kname):
    eng = ag.engine()
    D, N = 3, 700
    k = kernel(ag, cr.SE, cr.T_ARD, D)[0] if kname == "se_ard" else KERNELS["ard"](ag, D)
    X, y = data(N, D, dtype, seed=5)
    post = _handle(ag, k, X, y)
    h = post.data.C.h
    L = int(eng.L.agp_post_grad_len(h))
    outs = []
    for _ in range(2):
        g, nd, xg = np.zeros(L), np.empty(N, dtype=dtype), np.empty((D, N), dtype=dtype, order="F")
        eng.check(eng.L.agp_post_logpdf_grad_x(h, g.ctypes.data_as(C.POINTER(C.c_double)), ag._cabi.ptr(nd), 0, ag._cabi.ptr(xg)))
        outs.append((g, nd, xg))
    assert outs[0][2].tobytes() == outs[1][2].tobytes()
    g0, nd0 = np.zeros(L), np.empty(N, dtype=dtype)
    eng.check(eng.L.agp_post_logpdf_grad(h, g0.ctypes.data_as(C.POINTER(C.c_double)), ag._cabi.ptr(nd0)))
    # the per-point noise gradient is written element by element: the same bits.  The scalar sums leave their CTAs
    # through fp64 atomics, whose order varies from run to run in either entry point: equal to rounding.
    assert nd0.tobytes() == outs[0][1].tobytes()
    np.testing.assert_allclose(outs[0][0], g0, rtol=1e-12, atol=1e-12 * np.abs(g0).max())
    # the feature-major layout is the transpose of the point-major one, bit for bit; NULL outputs are skipped
    xf = np.empty((N, D), dtype=dtype, order="F")
    eng.check(eng.L.agp_post_logpdf_grad_x(h, None, None, 1, ag._cabi.ptr(xf)))
    assert xf.tobytes(order="F") == np.asfortranarray(outs[0][2].T).tobytes(order="F")


def test_device_memory_output(ag):
    torch = pytest.importorskip("torch")
    eng = ag.engine()
    D, N = 4, 500
    k = kernel(ag, cr.MATERN52, cr.T_SCALE, D)[0]
    X, y = data(N, D, np.float64, seed=6)
    post = _handle(ag, k, X, y)
    h = post.data.C.h
    ref_x = np.empty((D, N), order="F")
    eng.check(eng.L.agp_post_logpdf_grad_x(h, None, None, 0, ag._cabi.ptr(ref_x)))
    out = torch.empty((N, D), dtype=torch.float64, device="cuda")  # point-major D x N column-major == N x D row-major
    torch.cuda.synchronize()
    eng.set_memspace(ag._cabi.AGP_MEM_DEVICE)
    try:
        eng.check(eng.L.agp_post_logpdf_grad_x(h, None, None, 0, ag._cabi.ptr(out.data_ptr())))
    finally:
        eng.set_memspace(ag._cabi.AGP_MEM_HOST)
    assert out.cpu().numpy().tobytes() == ref_x.tobytes(order="F")


def test_errors(ag):
    cabi = ag._cabi
    eng = ag.engine()
    X, y = data(80, 2, np.float64, seed=7)
    post = _handle(ag, ag.SqExponentialKernel(), X, y)
    xg = np.empty((2, 80), order="F")
    assert eng.L.agp_post_logpdf_grad_x(post.data.C.h, None, None, 2, cabi.ptr(xg)) == cabi.AGP_ERR_INVALID
    X2, y2 = data(20, 2, np.float64, seed=8)
    p2 = ag.posterior(post(ag.RowVecs(X2), 0.1), y2)
    xg2 = np.empty((2, 100), order="F")
    assert eng.L.agp_post_logpdf_grad_x(p2.data.C.h, None, None, 0, cabi.ptr(xg2)) == cabi.AGP_ERR_UNSUPPORTED
    # the first handle still works
    eng.check(eng.L.agp_post_logpdf_grad_x(post.data.C.h, None, None, 0, cabi.ptr(xg)))


def test_reference_input_gradient_replay(ag):
    """test/finite_gp_projection.jl:162-173: SE, f(x, 1e-3), y = ones, against torch fp64 autograd"""
    torch = pytest.importorskip("torch")
    from test_grad_x_model import torch_logpdf
    x = np.random.default_rng(123).standard_normal(11)
    lp, g = ag.logpdf_grad(ag.GP(ag.SqExponentialKernel())(x, 1e-3), np.ones(11), inputs=True)
    xt = torch.tensor(x[:, None], dtype=torch.float64, requires_grad=True)
    torch_logpdf(torch, ref.KernelSpec(cr.SE), xt, np.ones(11), 1e-3, 0.0).backward()
    want = xt.grad.numpy()[:, 0]
    np.testing.assert_allclose(g["x"], want, rtol=1e-7, atol=1e-7 * np.abs(want).max())


def test_deep_kernel_learning_replay(ag):
    """a seeded MLP maps 1-D inputs to 2-D features, loss = -logpdf of an SE GP on the features; the device gradient
    enters the network through features.backward(g) and must equal pure torch fp64 autograd; ten gradient steps lower
    the loss"""
    torch = pytest.importorskip("torch")
    from test_grad_x_model import torch_logpdf
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    N = 120
    x = torch.tensor(rng.uniform(-3, 3, (N, 1)), dtype=torch.float64)
    y = np.sinc(x.numpy()[:, 0]) + 0.01 * rng.standard_normal(N)
    net = torch.nn.Sequential(torch.nn.Linear(1, 20), torch.nn.Tanh(), torch.nn.Linear(20, 2)).double()
    s2 = 0.01 ** 2 + 1e-3

    def device_step():
        net.zero_grad()
        feats = net(x)
        F = feats.detach().numpy()
        lp, g = ag.logpdf_grad(ag.GP(ag.SqExponentialKernel())(ag.RowVecs(F), s2), y, inputs=True)
        feats.backward(torch.from_numpy(-g["x"]))  # loss = -logpdf
        return -lp, [p.grad.clone() for p in net.parameters()]

    loss0, grads = device_step()
    net.zero_grad()
    (-torch_logpdf(torch, ref.KernelSpec(cr.SE), net(x), y, s2, 0.0)).backward()
    gts = [p.grad for p in net.parameters()]
    # the last bias's gradient is sum_i dL/dx_i, 0 up to rounding for a stationary kernel: the scale is the whole gradient's
    scale = max(gt.abs().max().item() for gt in gts)
    for gd, gt in zip(grads, gts):
        np.testing.assert_allclose(gd.numpy(), gt.numpy(), rtol=1e-7, atol=1e-7 * scale)
    lr = 1e-2 / np.sqrt(sum(float((g_ * g_).sum()) for g_ in grads))  # one fixed step size for all ten steps
    for step in range(10):
        if step:
            _, grads = device_step()
        with torch.no_grad():
            for p, gp in zip(net.parameters(), grads):
                p -= lr * gp
    loss, _ = device_step()
    assert loss < loss0, (loss, loss0)
