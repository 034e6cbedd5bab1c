"""The gradient of the VFE objectives with respect to the training inputs on the device (agp_vfe_elbo_grad_x through
approx_log_evidence_grad / elbo_grad with inputs=True) against the NumPy model tests/vfe_grad_x_ref.py (pinned to torch
fp64 autograd by tests/test_vfe_grad_x_model.py): every family x transform x dtype on test_gpu_vfe_grad.py's small cases
in the row, column and vector containers; the sizes where G = R K_zx comes from the int8-slice product; forced chunkings;
translation invariance; agreement with agp_vfe_elbo_grad, determinism, permutation of the data; launches and device
memory; device-memory outputs; errors; and a sparse deep-kernel-learning replay through a torch network.

Tolerance: fp64 rtol 1e-7, fp32 rtol 2e-2 (against the model on the fp32-rounded inputs), atol the same times x_scale,
the larger of the two terms x sums (the K_zx part and, for the Linear kernel, the kdiag part).  No case needs more: the
degenerate Linear case that z needs rtol 1e-5 for (D = 1, M = 128, K_zz of rank 2 plus jitter) stays at 1.6e-11 of
x_scale.  Measured worst errors (H100, in units of x_scale): fp64 9.3e-11 on the small cases and 4.5e-11 at M = 2304;
fp32 5.8e-8 (the fp64 result rounded to fp32)."""
import ctypes as C

import numpy as np
import pytest

import vfe_grad_x_ref as vx
from oracle import agp_ref as ref
from test_gpu_vfe_grad import FAMILIES, Problem

pytestmark = pytest.mark.gpu
RT = {np.float64: 1e-7, np.float32: 2e-2}


class XProblem(Problem):
    """Problem with a vector container for D = 1 and the input gradient"""

    def wrap(self, A):
        if self.container == "vec":
            return A[:, 0].copy()
        return super().wrap(A)

    def device_x(self, objective=0, inputs=True):
        fz, fx = self.args()
        vfe = self.ag.VFE(fz) if objective == 0 else self.ag.DTC(fz)
        v, g = self.ag.approx_log_evidence_grad(vfe, fx, self.y, inputs=inputs)
        return float(v), g

    def as_nd(self, x):
        """the device's x in the container's shape -> N x D"""
        return {"row": lambda: x, "col": lambda: x.T, "vec": lambda: x[:, None]}[self.container]()

    def model_x(self, objective=0):
        return vx.vfe_grad_x(self.k, self.mean_ref, self.noise_ref, self.X.astype(np.float64), self.y.astype(np.float64),
                             self.Z.astype(np.float64), ref.NoiseSpec(0, self.jit), objective)


def check_x(p, objective, label=""):
    """returns the worst error in units of x_scale"""
    v, g = p.device_x(objective)
    x = p.as_nd(g["x"])
    assert g["x"].dtype == p.dtype and np.all(np.isfinite(x)), label
    want, xs = p.model_x(objective)
    rtol = RT[p.dtype]
    np.testing.assert_allclose(x.astype(np.float64), want, rtol=rtol, atol=rtol * xs, err_msg=str(label))
    return float(np.max(np.abs(x.astype(np.float64) - want))) / xs


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform", [ref.T_NONE, ref.T_SCALE, ref.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_matches_model_small(ag, family, transform, dtype):
    cases = [(333, 7, 1, "vec", 0, 0, 0), (333, 128, 5, "col", 1, 2, 1), (3000, 7, 5, "row", 1, 1, 0),
             (3000, 128, 1, "col", 0, 1, 1), (3000, 375, 40, "row", 1, 2, 0), (333, 375, 40, "col", 0, 0, 1)]
    for i, (N, M, D, container, nk, mk, obj) in enumerate(cases):
        p = XProblem(ag, family, transform, N, M, D, dtype, nk, mk, container, seed=i)
        w = check_x(p, obj, label=(N, M, D, container, nk, mk, obj))
        print("worst x", np.dtype(dtype).name, family, transform, (N, M, D), "%.3g" % w)


@pytest.mark.parametrize("N,M,dtype", [(3000, 1100, np.float64), (6000, 2304, np.float64), (20000, 1100, np.float32),
                                       (20000, 4224, np.float32)])
def test_matches_model_tensor_sizes(ag, N, M, dtype):
    """G = R K_zx on the int8-slice product (M >= 1024), with the tensor forward substitution at M = 2304"""
    p = XProblem(ag, ref.SE, ref.T_SCALE, N, M, 8, dtype, noise_kind=1, mean_kind=1)
    w = check_x(p, 0)
    print("worst x", np.dtype(dtype).name, "tensor", (N, M), "%.3g" % w)


def test_forced_chunks_agree_with_one_chunk(ag, monkeypatch):
    p = XProblem(ag, ref.MATERN32, ref.T_ARD, 3000, 1100, 6, np.float64, noise_kind=1, mean_kind=2)
    _, g1 = p.device_x(0)
    for chunk in ("128", "1024", "1152"):
        monkeypatch.setenv("AGP_VFE_CHUNK", chunk)
        _, g = p.device_x(0)
        np.testing.assert_allclose(g["x"], g1["x"], rtol=1e-10, atol=1e-10 * np.abs(g1["x"]).max(), err_msg=chunk)


@pytest.mark.parametrize("family", [ref.SE, ref.MATERN12, ref.MATERN32, ref.MATERN52])
def test_translation_invariance(ag, family):
    """stationary kernel: shifting every x and z by the same vector leaves the objective unchanged, so
    sum_n xbar_n + sum_m zbar_m = 0 up to rounding (no model involved)"""
    p = XProblem(ag, family, ref.T_ARD, 2000, 150, 3, np.float64, noise_kind=1, mean_kind=1)
    for objective in (0, 1):
        _, g = p.device_x(objective)
        x, z = g["x"], g["z"]
        tot = x.sum(0) + z.sum(0)
        assert np.all(np.abs(tot) <= 1e-10 * (np.abs(x).sum(0) + np.abs(z).sum(0))), (objective, tot)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_agreement_determinism_and_permutation(ag, dtype):
    p = XProblem(ag, ref.MATERN52, ref.T_SCALE, 1500, 90, 2, dtype, noise_kind=1, mean_kind=2)
    v0, g0 = p.device_x(0, inputs=False)
    v1, g1 = p.device_x(0)
    v2, g2 = p.device_x(0)
    assert set(g1) == set(g0) | {"x"}
    for key in ("z", "noise", "mean_v"):  # summed in a fixed order: bit for bit
        assert np.asarray(g1[key]).tobytes() == np.asarray(g0[key]).tobytes(), key
    for key in ("variance", "scale"):  # fp64 atomics: to rounding
        assert abs(g1[key] - g0[key]) <= 1e-12 * abs(g0[key]), key
    assert abs(v1 - v0) <= 1e-6 * abs(v0)
    assert g1["x"].tobytes() == g2["x"].tobytes()
    perm = np.random.default_rng(1).permutation(1500)
    p.X, p.y, p.s2 = p.X[perm].copy(), p.y[perm].copy(), p.s2[perm].copy()  # the CustomMean follows the points
    _, gp = p.device_x(0)
    tol = 1e-9 if dtype == np.float64 else 1e-5
    np.testing.assert_allclose(gp["x"], g1["x"][perm], rtol=tol, atol=tol * np.abs(g1["x"]).max())


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_launches_and_memory(ag, monkeypatch, dtype):
    """inputs=True adds two launches per chunk of the streamed pass (vfe_x_grad_kernel and vfe_x_finish_kernel) and
    nothing else; device memory comes back"""
    torch = pytest.importorskip("torch")
    eng = ag.engine()
    p = XProblem(ag, ref.SE, ref.T_ARD, 3000, 200, 3, dtype, noise_kind=1, mean_kind=2)

    def launches(inputs):
        l0 = eng.launch_count()
        p.device_x(0, inputs=inputs)
        return eng.launch_count() - l0

    for chunk, nchunks in ((None, 1), ("1024", 3), ("128", 24)):
        if chunk:
            monkeypatch.setenv("AGP_VFE_CHUNK", chunk)
        base = launches(False)
        assert launches(False) == base
        assert launches(True) - base == 2 * nchunks, (chunk, base)
    monkeypatch.delenv("AGP_VFE_CHUNK")
    p.device_x(0)
    free0 = torch.cuda.mem_get_info()[0]
    p.device_x(0)
    assert abs(torch.cuda.mem_get_info()[0] - free0) <= 64 << 20


def _raw_args(ag, p, objective=0, kernel=None):
    fz, fx = p.args()
    f, dt, pts, z, y, ks, ms, ns, js, keep = ag.api._vfe_args(ag.VFE(fz), fx, p.y)
    if kernel is not None:
        ks = ag.api._kernel_struct(kernel, dt, keep, D=pts.D)
    return dt, pts, z, y, ks, ms, ns, js, keep


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_device_memory_outputs(ag, dtype):
    """under AGP_MEM_DEVICE with torch buffers (X, Z, y in, every array out) x is bit-identical to the host result, in
    both layouts"""
    torch = pytest.importorskip("torch")
    cabi = ag._cabi
    eng = ag.engine()
    p = XProblem(ag, ref.MATERN32, ref.T_ARD, 700, 60, 3, dtype, noise_kind=1, mean_kind=2)
    dt, pts, z, y, ks, ms, ns, js, keep = _raw_args(ag, p)
    N, M, D = pts.n, z.n, pts.D
    tdt = torch.float64 if dt == np.float64 else torch.float32
    for layout in (cabi.AGP_POINT_MAJOR, cabi.AGP_FEATURE_MAJOR):
        Xh = pts.a if layout == 0 else np.asfortranarray(pts.a.reshape(N, D))
        Zh = z.a if layout == 0 else np.asfortranarray(z.a.reshape(M, D))
        g = np.zeros(5 + D)
        xh = np.empty(N * D, dtype=dt)
        v = np.empty(1, dtype=dt)
        eng.check(eng.L.agp_vfe_elbo_grad_x(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), layout,
                                            cabi.ptr(Xh), N, D, cabi.ptr(Zh), M, C.byref(js), cabi.ptr(y), 0, cabi.ptr(v),
                                            g.ctypes.data_as(C.POINTER(C.c_double)), None, None, None, cabi.ptr(xh)))
        Xd = torch.from_numpy(np.ravel(Xh, order="K").copy()).cuda()
        Zd = torch.from_numpy(np.ravel(Zh, order="K").copy()).cuda()
        yd = torch.from_numpy(np.asarray(y)).cuda()
        xd = torch.empty(N * D, dtype=tdt, device="cuda")
        ndd = torch.empty(N, dtype=tdt, device="cuda")
        zd = torch.empty(M * D, dtype=tdt, device="cuda")
        gd = np.zeros(5 + D)
        torch.cuda.synchronize()
        eng.set_memspace(cabi.AGP_MEM_DEVICE)
        try:
            eng.check(eng.L.agp_vfe_elbo_grad_x(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), layout,
                                                cabi.ptr(Xd.data_ptr()), N, D, cabi.ptr(Zd.data_ptr()), M, C.byref(js),
                                                cabi.ptr(yd.data_ptr()), 0, None, gd.ctypes.data_as(C.POINTER(C.c_double)),
                                                cabi.ptr(ndd.data_ptr()), None, cabi.ptr(zd.data_ptr()),
                                                cabi.ptr(xd.data_ptr())))
        finally:
            eng.set_memspace(cabi.AGP_MEM_HOST)
        assert xd.cpu().numpy().tobytes() == xh.tobytes(), layout
        if layout == 1:  # the feature-major layout is the transpose of the point-major one
            assert np.array_equal(xh.reshape(D, N).T, x0.reshape(N, D))
        x0 = xh.copy()


def test_errors_and_reuse(ag):
    cabi = ag._cabi
    eng = ag.engine()
    p = XProblem(ag, ref.SE, ref.T_NONE, 400, 20, 2, np.float64)

    def call(objective=0, layout=0, kernel=None):
        dt, pts, z, y, ks, ms, ns, js, keep = _raw_args(ag, p, objective, kernel)
        v = np.empty(1)
        g = np.zeros(5 + pts.D)
        xg = np.empty((pts.n, pts.D))
        return eng.L.agp_vfe_elbo_grad_x(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), layout,
                                         cabi.ptr(pts.a), pts.n, pts.D, cabi.ptr(z.a), z.n, C.byref(js), cabi.ptr(y),
                                         objective, cabi.ptr(v), g.ctypes.data_as(C.POINTER(C.c_double)), None, None, None,
                                         cabi.ptr(xg))

    assert call(layout=5) == cabi.AGP_ERR_INVALID
    assert call(objective=2) == cabi.AGP_ERR_INVALID
    assert call(kernel=ag.SqExponentialKernel() + ag.Matern32Kernel()) == cabi.AGP_ERR_UNSUPPORTED
    # non-PD K_zz at M = 1100: every inducing point twice, no jitter
    q = XProblem(ag, ref.SE, ref.T_NONE, 3000, 550, 2, np.float64)
    Zd = np.concatenate([q.Z, q.Z])
    f = ag.GP(q.kern)
    with pytest.raises(ag.PosDefException) as e:
        ag.elbo_grad(ag.VFE(f(ag.RowVecs(Zd), 0.0)), f(ag.RowVecs(q.X), 0.1), q.y, inputs=True)
    assert e.value.code == cabi.AGP_ERR_NOT_POSDEF and e.value.info != 0
    assert call() == cabi.AGP_OK
    check_x(p, 0)


def test_sparse_deep_kernel_learning_replay(ag):
    """a seeded MLP maps 1-D inputs to 2-D features, loss = -elbo of an SE sparse GP (N = 2000, M = 32) on the features;
    the device gradient enters the network through feats.backward(-g["x"]) and must equal pure torch fp64 autograd of
    the dense restatement of the elbo; ten fixed-size gradient steps lower the loss"""
    torch = pytest.importorskip("torch")
    from test_vfe_grad_model import torch_objective
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    N, M = 2000, 32
    x = torch.tensor(rng.uniform(-3, 3, (N, 1)), dtype=torch.float64)
    y = np.sinc(x.numpy()[:, 0]) + 0.05 * rng.standard_normal(N)
    net = torch.nn.Sequential(torch.nn.Linear(1, 20), torch.nn.Tanh(), torch.nn.Linear(20, 2)).double()
    with torch.no_grad():
        Z = net(torch.linspace(-3, 3, M, dtype=torch.float64)[:, None]).numpy().copy()
    s2, jit = 0.05 ** 2, 1e-4
    f = ag.GP(ag.SqExponentialKernel())

    def device_step():
        net.zero_grad()
        feats = net(x)
        v, g = ag.elbo_grad(ag.VFE(f(ag.RowVecs(Z), jit)), f(ag.RowVecs(feats.detach().numpy()), s2), y, inputs=True)
        feats.backward(torch.from_numpy(-g["x"]))  # loss = -elbo
        return -v, [q.grad.clone() for q in net.parameters()]

    loss0, grads = device_step()
    net.zero_grad()
    ones = torch.ones(2, dtype=torch.float64)
    fo = torch_objective(torch, ref.SE, 1.0, ones, 0.0, net(x), torch.from_numpy(Z), y, torch.tensor(s2, dtype=torch.float64),
                         torch.zeros(N, dtype=torch.float64), jit, 0)
    (-fo).backward()
    assert abs(-fo.item() - loss0) <= 1e-9 * abs(loss0)
    gts = [q.grad for q in net.parameters()]
    scale = max(gt.abs().max().item() for gt in gts)
    for gd, gt in zip(grads, gts):
        np.testing.assert_allclose(gd.numpy(), gt.numpy(), rtol=1e-7, atol=1e-7 * scale)
    lr = 1e-2 / np.sqrt(sum(float((g_ * g_).sum()) for g_ in grads))  # one fixed step size for all ten steps
    for step in range(10):
        if step:
            _, grads = device_step()
        with torch.no_grad():
            for q, gq in zip(net.parameters(), grads):
                q -= lr * gq
    loss, _ = device_step()
    assert loss < loss0, (loss, loss0)
