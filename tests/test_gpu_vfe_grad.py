"""The gradient of the VFE objectives on the device (agp_vfe_elbo_grad through approx_log_evidence_grad / elbo_grad)
against the NumPy model tests/vfe_grad_ref.py (itself pinned to torch fp64 autograd by tests/test_vfe_grad_model.py):
every family x transform x dtype at small sizes in both point containers with per-point noise, vector means and both
objectives; the sizes where the passes run on the tensor cores (int8-slice products in both passes at M = 1100, tensor
forward substitution at M = 2304, fp32 at M = 4224), each branch asserted from the launch counter, and forced chunkings;
the invariants (the value is agp_vfe_elbo's, agp_vfe_elbo's launches are unchanged,
deterministic per-point and inducing-point outputs, device memory, error codes, permutation of the data); and a training
replay with scipy's L-BFGS-B driven by the device gradient.

Tolerance: fp64 rtol 1e-7, fp32 rtol 2e-2 (against the model on the fp32-rounded inputs), atol the same times max|g| over the hyper-parameter entries, and for z times the larger of its two
summed terms (K_zz and K_zx parts), which cancel to a much smaller gradient for the Linear kernel.  One configuration
gets z_rtol 1e-5, stated in the test: the Linear kernel at D = 1 with M = 128 inducing points, where K_zz has rank 2 plus
jitter and z is ~1e8 times smaller than its terms (measured: 6e-7 of the larger term, N = 3000, DTC).  Inputs keep
cond(K_zz + J) <= 1e4: the jitter is raised to lambda_max(K_zz) / 1e4 where the points alone do not.

An fp32 problem takes its value from the fp32 pass (agp_vfe_elbo's) and its gradient from fp64 on the same problem:
formed entirely in fp32 the gradient missed the model by far more than rtol 2e-2 (worst z entry off by 0.39 where max|z|
was 0.18; SE, N = 3000, M = 128, D = 1, cond(K_zz + J) <= 1e4), the adjoints being differences of terms about 1e5 times
larger than the result.  Measured worst error of the fp32 cases (H100, in units of each
entry's atol scale, so rtol 2e-2 allows 2e-2): 7.7e-7, the degenerate Linear case below; 8.7e-8 at M = 4224, N = 20 000."""
import numpy as np
import pytest

import vfe_grad_ref as vg
from oracle import agp_ref as ref

pytestmark = pytest.mark.gpu

FAMILIES = [ref.SE, ref.MATERN12, ref.MATERN32, ref.MATERN52, ref.LINEAR]
AG_FAMILY = {ref.SE: "SqExponentialKernel", ref.MATERN12: "Matern12Kernel", ref.MATERN32: "Matern32Kernel",
             ref.MATERN52: "Matern52Kernel"}


class Problem:
    def __init__(self, ag, family, transform, N, M, D, dtype, noise_kind=0, mean_kind=0, container="row", seed=0):
        rng = np.random.default_rng(seed + 1000 * family + 100 * transform + N + M + D)
        self.ag, self.dtype, self.container = ag, dtype, container
        self.X = (rng.uniform(-2, 2, (N, D)) / np.sqrt(D)).astype(dtype)
        self.Z = (rng.uniform(-2, 2, (M, D)) / np.sqrt(D)).astype(dtype)
        self.y = (np.sin(2.0 * self.X.astype(np.float64)).sum(1) + 0.1 * rng.normal(size=N)).astype(dtype)
        ard = rng.uniform(0.6, 1.4, D).astype(dtype) if transform == ref.T_ARD else None
        var, sc, lc = 1.3, 0.8, 0.4
        self.k = ref.KernelSpec(family, var, transform, scale=sc, ard=None if ard is None else ard.astype(np.float64),
                                linear_c=lc if family == ref.LINEAR else 0.0)
        base = ag.LinearKernel(lc) if family == ref.LINEAR else getattr(ag, AG_FAMILY[family])()
        if transform == ref.T_SCALE:
            base = base.compose(ag.ScaleTransform(sc))
        elif transform == ref.T_ARD:
            base = base.compose(ag.ARDTransform(ard))
        self.kern = var * base
        Kzz = ref.kernelmatrix(self.k, self.Z.astype(np.float64))
        self.jit = float(max(1e-6 if dtype == np.float64 else 1e-4, np.linalg.eigvalsh(Kzz)[-1] / 1e4))
        if noise_kind == 0:
            self.s2, self.noise_ref = 0.1, ref.NoiseSpec(0, 0.1)
        else:
            self.s2 = rng.uniform(0.05, 0.3, N).astype(dtype)
            self.noise_ref = ref.NoiseSpec(1, v=self.s2.astype(np.float64))
        self.mean_ag, self.mean_ref = None, ref.MeanSpec()
        if mean_kind == 1:
            self.mean_ag, self.mean_ref = 0.3, ref.MeanSpec(1, 0.3)
        elif mean_kind == 2:
            def mfn(xi):
                return 0.2 * np.cos(3.0 * float(np.ravel(xi)[0]))
            self.mean_ag = ag.CustomMean(mfn)
            self.mean_ref = ref.MeanSpec(2, v=np.array([mfn(xi) for xi in self.X], dtype=dtype).astype(np.float64))

    def wrap(self, A):
        return self.ag.RowVecs(A) if self.container == "row" else self.ag.ColVecs(A.T.copy())

    def args(self):
        ag = self.ag
        f = ag.GP(self.kern) if self.mean_ag is None else ag.GP(self.mean_ag, self.kern)
        return f(self.wrap(self.Z), self.jit), f(self.wrap(self.X), self.s2)

    def device(self, objective=0):
        fz, fx = self.args()
        vfe = self.ag.VFE(fz) if objective == 0 else self.ag.DTC(fz)
        v, g = self.ag.approx_log_evidence_grad(vfe, fx, self.y)
        assert g["z"].dtype == self.dtype
        g = dict(g)
        g["z"] = g["z"] if self.container == "row" else g["z"].T
        return float(v), g

    def model(self, objective=0):
        v, g, z, zs = vg.vfe_grad(self.k, self.mean_ref, self.noise_ref, self.X.astype(np.float64),
                                  self.y.astype(np.float64), self.Z.astype(np.float64), ref.NoiseSpec(0, self.jit), objective,
                                  z_scale=True)
        g["z"] = z
        self.z_scale = zs
        return v, g


def assert_close(dev, want, z_scale, label="", z_rtol=1e-7, dtype=np.float64):
    """returns the worst gradient error in units of its atol scale"""
    rtol = 1e-7 if dtype == np.float64 else 2e-2
    z_rtol = z_rtol if dtype == np.float64 else rtol
    (v, g), (vm, gm) = dev, want
    assert abs(v - vm) <= rtol * max(1.0, abs(vm)), (label, v, vm)
    worst = 0.0
    assert g.keys() == gm.keys(), (label, g.keys(), gm.keys())
    hyper = max(np.abs(np.atleast_1d(gm[k])).max() for k in gm if k != "z")
    for key in gm:
        r = z_rtol if key == "z" else rtol
        scale = z_scale if key == "z" else hyper
        np.testing.assert_allclose(np.asarray(g[key], dtype=np.float64), gm[key], rtol=r, atol=r * scale,
                                   err_msg="%s %s" % (label, key))
        worst = max(worst, float(np.max(np.abs(np.asarray(g[key], dtype=np.float64) - gm[key]))) / scale)
    return worst


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform", [ref.T_NONE, ref.T_SCALE, ref.T_ARD])
@pytest.mark.parametrize("family", FAMILIES)
def test_matches_model_small(ag, family, transform, dtype):
    cases = [(333, 7, 1, "row", 0, 0, 0), (333, 128, 5, "col", 1, 2, 1), (3000, 7, 5, "row", 1, 1, 0),
             (3000, 128, 1, "col", 0, 1, 1), (3000, 375, 40, "row", 1, 2, 0), (333, 375, 40, "col", 0, 0, 1)]
    for i, (N, M, D, container, nk, mk, obj) in enumerate(cases):
        p = Problem(ag, family, transform, N, M, D, dtype, nk, mk, container, seed=i)
        want = p.model(obj)
        degenerate = family == ref.LINEAR and D == 1 and M == 128  # K_zz: rank 2 plus jitter
        w = assert_close(p.device(obj), want, p.z_scale, label=(N, M, D, container, nk, mk, obj),
                         z_rtol=1e-5 if degenerate else 1e-7, dtype=dtype)
        print("worst", np.dtype(dtype).name, family, transform, (N, M, D), "%.3g" % w)


@pytest.mark.parametrize("N,M,dtype", [(3000, 1100, np.float64), (6000, 2304, np.float64), (3000, 1100, np.float32),
                                       (20000, 4224, np.float32)])
def test_matches_model_tensor_sizes(ag, N, M, dtype):
    """M = 1100: both passes use the int8-slice products; M = 2304: V_z and V_m come from the tensor forward substitution
    as well; fp32 M = 4224, N = 20 000: the C5 shape scaled, its pass 1 on the fp32 int8-slice Cholesky"""
    p = Problem(ag, ref.SE, ref.T_SCALE, N, M, 8, dtype, noise_kind=1, mean_kind=1)
    want = p.model(0)
    w = assert_close(p.device(0), want, p.z_scale, dtype=dtype)
    print("worst", np.dtype(dtype).name, "tensor", (N, M), "%.3g" % w)


@pytest.mark.parametrize("M,branch", [(1100, "int8"), (2304, "int8"), (375, "tile")])
def test_branch_from_launch_counter(ag, M, branch):
    """launches of the gradient beyond those of the elbo pass, under the automatic policy and with the tile kernels
    forced (fp64_mode 0): at M = 1100 only G = R K_zx differs (int8-slice product: slices of R once, then per chunk the
    slices of K_zx and the update, against one tile GEMM), at M = 2304 the forward substitutions on the identity as well,
    below m_pad = 1024 nothing does"""
    eng = ag.engine()
    p = Problem(ag, ref.SE, ref.T_SCALE, 3000, M, 4, np.float64)

    def extra():
        fz, fx = p.args()
        vfe = ag.VFE(fz)
        l0 = eng.launch_count()
        ag.approx_log_evidence(vfe, fx, p.y)
        l1 = eng.launch_count()
        ag.approx_log_evidence_grad(vfe, fx, p.y)
        return (eng.launch_count() - l1) - (l1 - l0)

    auto = extra()
    old = eng.get_config().fp64_mode
    eng.set_config(fp64_mode=0)
    try:
        tile = extra()
    finally:
        eng.set_config(fp64_mode=old)
    if M == 1100:
        # 3000 points, one chunk: row scales + slices of R, row scales + slices of K_zx and the update, for 1 tile GEMM
        assert auto == tile + 4, (auto, tile)
    elif branch == "int8":
        assert auto != tile, (auto, tile)
    else:
        assert auto == tile, (auto, tile)


def test_forced_chunks_agree_with_one_chunk(ag, monkeypatch):
    p = Problem(ag, ref.MATERN32, ref.T_ARD, 3000, 1100, 6, np.float64, noise_kind=1, mean_kind=2)
    v1, g1 = p.device(0)
    tol = 1e-10
    for chunk in ("1024", "1152", "128"):
        monkeypatch.setenv("AGP_VFE_CHUNK", chunk)
        v, g = p.device(0)
        assert abs(v - v1) <= tol * abs(v1), chunk
        for key in g1:
            a, b = np.asarray(g[key], np.float64), np.asarray(g1[key], np.float64)
            np.testing.assert_allclose(a, b, rtol=tol, atol=tol * np.abs(b).max(), err_msg="%s %s" % (chunk, key))


@pytest.mark.parametrize("objective", [0, 1])
def test_value_launches_determinism_and_memory(ag, objective):
    torch = pytest.importorskip("torch")
    eng = ag.engine()
    p = Problem(ag, ref.SE, ref.T_ARD, 2000, 200, 3, np.float64, noise_kind=1, mean_kind=2)
    fz, fx = p.args()
    vfe = ag.VFE(fz) if objective == 0 else ag.DTC(fz)
    l0 = eng.launch_count()
    e0 = ag.approx_log_evidence(vfe, fx, p.y, return_dtc=True)
    n_elbo = eng.launch_count() - l0
    free0 = torch.cuda.mem_get_info()[0]
    v, g = ag.approx_log_evidence_grad(vfe, fx, p.y)
    v2, g2 = ag.approx_log_evidence_grad(vfe, fx, p.y)
    # the value is the one the same pass gives agp_vfe_elbo (its scalars are summed with fp64 atomics)
    assert abs(v - e0[objective]) <= 1e-13 * abs(e0[objective])
    for key in ("z", "noise", "mean_v"):
        assert np.asarray(g[key]).tobytes() == np.asarray(g2[key]).tobytes(), key
    l1 = eng.launch_count()
    ag.approx_log_evidence(vfe, fx, p.y, return_dtc=True)
    assert eng.launch_count() - l1 == n_elbo
    assert abs(torch.cuda.mem_get_info()[0] - free0) <= 64 << 20


def test_permutation_of_the_data(ag):
    p = Problem(ag, ref.MATERN52, ref.T_SCALE, 1500, 90, 2, np.float64, noise_kind=1, mean_kind=1)
    v, g = p.device(0)
    perm = np.random.default_rng(1).permutation(1500)
    p.X, p.y, p.s2 = p.X[perm].copy(), p.y[perm].copy(), p.s2[perm].copy()
    vp, gp = p.device(0)
    assert abs(v - vp) <= 1e-10 * abs(v)
    for key in ("variance", "scale", "mean_c", "z"):
        np.testing.assert_allclose(gp[key], g[key], rtol=1e-9, atol=1e-9 * np.abs(g[key]).max())
    np.testing.assert_allclose(gp["noise"], g["noise"][perm], rtol=1e-9, atol=1e-12)


def test_errors_and_reuse(ag):
    cabi = ag._cabi
    eng = ag.engine()
    p = Problem(ag, ref.SE, ref.T_NONE, 400, 20, 2, np.float64)
    fz, fx = p.args()

    def call(objective=0, layout=0, kernel=None, fz_=fz):
        import ctypes as C
        f, dt, pts, z, y, ks, ms, ns, js, keep = ag.api._vfe_args(ag.VFE(fz_), fx, p.y)
        if kernel is not None:
            ks = ag.api._kernel_struct(kernel, dt, keep, D=pts.D)
        v = np.empty(1)
        g = np.zeros(5 + pts.D)
        zg = np.empty((z.n, pts.D))
        return eng.L.agp_vfe_elbo_grad(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), layout,
                                       cabi.ptr(pts.a), pts.n, pts.D, cabi.ptr(z.a), z.n, C.byref(js), cabi.ptr(y), objective,
                                       cabi.ptr(v), g.ctypes.data_as(C.POINTER(C.c_double)), None, None, cabi.ptr(zg))

    assert call(objective=2) == cabi.AGP_ERR_INVALID
    assert call(layout=5) == cabi.AGP_ERR_INVALID
    assert call(kernel=ag.SqExponentialKernel() + ag.Matern32Kernel()) == cabi.AGP_ERR_UNSUPPORTED
    # non-PD K_zz at M = 1100: every inducing point twice, no jitter
    q = Problem(ag, ref.SE, ref.T_NONE, 3000, 550, 2, np.float64)
    Zd = np.concatenate([q.Z, q.Z])
    f = ag.GP(q.kern)
    with pytest.raises(ag.PosDefException) as e:
        ag.elbo_grad(ag.VFE(f(ag.RowVecs(Zd), 0.0)), f(ag.RowVecs(q.X), 0.1), q.y)
    assert e.value.code == cabi.AGP_ERR_NOT_POSDEF and e.value.info != 0
    assert eng.L.agp_last_info(eng.h) == e.value.info
    assert call() == cabi.AGP_OK
    want = p.model(0)
    assert_close(p.device(0), want, p.z_scale)


def test_training_replay_lbfgs(ag):
    """a 1-D sparse regression (N = 2000, M = 32): L-BFGS-B over log sigma_f^2, log lengthscale, log sigma^2 and z on the
    negative elbo, once with the device gradient and once with the model's; the accepted steps decrease the objective
    and both runs end at the same optimum"""
    from scipy.optimize import minimize
    rng = np.random.default_rng(0)
    N, M = 2000, 32
    x = np.sort(rng.uniform(-3, 3, N))
    y = np.sin(2 * x) + 0.3 * np.cos(5 * x) + 0.1 * rng.normal(size=N)
    z0 = np.linspace(-2.5, 2.5, M)
    th0 = np.concatenate([[0.0, 0.0, np.log(0.1)], z0])
    jit = 1e-6

    def device(th):
        v, l, s2 = np.exp(th[:3])
        f = ag.GP(v * ag.with_lengthscale(ag.SqExponentialKernel(), l))
        val, g = ag.elbo_grad(ag.VFE(f(th[3:], jit)), f(x, s2), y)
        return val, np.concatenate([[v * g["variance"], -g["scale"] / l, s2 * g["noise"]], g["z"]])

    def model(th):
        v, l, s2 = np.exp(th[:3])
        k = ref.KernelSpec(ref.SE, v, ref.T_SCALE, scale=1.0 / l)
        val, g, zg = vg.vfe_grad(k, ref.MeanSpec(), ref.NoiseSpec(0, s2), x[:, None], y, th[3:, None], ref.NoiseSpec(0, jit))
        return val, np.concatenate([[v * g["variance"], -g["scale"] / l, s2 * g["noise"]], zg[:, 0]])

    results = []
    for fn in (device, model):
        trace = []

        def fun(th):
            val, g = fn(th)
            return -val, -g

        r = minimize(fun, th0, jac=True, method="L-BFGS-B", options={"maxiter": 60},
                     callback=lambda th: trace.append(fun(th)[0]))
        assert all(b <= a for a, b in zip(trace, trace[1:])), trace
        assert r.fun < fun(th0)[0] - 100.0
        results.append(r)
    rd, rm = results
    assert abs(rd.fun - rm.fun) <= 1e-6 * abs(rm.fun), (rd.fun, rm.fun)
