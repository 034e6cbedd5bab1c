"""The gradient of the VFE objectives (agp_vfe_elbo_grad) without a GPU: the NumPy model tests/vfe_grad_ref.py pinned
against torch fp64 autograd of an independent dense restatement of the elbo and DTC objectives, against central
differences and against the oracle's values; the Python mirror driven through a stand-in library; and ptxas on the new
kernels."""
import ctypes as C
import itertools
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import fake_libagp
import vfe_grad_ref as vg
from oracle import agp_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "abstractgps.jl_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
FAMILIES = [ref.SE, ref.MATERN12, ref.MATERN32, ref.MATERN52, ref.LINEAR]


# ---- an independent torch restatement: the dense N x N form of the bound ------------------------------------------------
def _torch_kernel(torch, family, var, t, c, A, B, same):
    At, Bt = A * t, B * t
    if family == ref.LINEAR:
        return var * (At @ Bt.T + c)
    diff = At[:, None, :] - Bt[None, :, :]
    d2 = (diff * diff).sum(2)
    if family == ref.SE:
        return var * torch.exp(-0.5 * d2)
    pos = d2 > 0  # coincident points: kappa = 1 with a zero derivative (the Matern 1/2 subgradient the device uses)
    d = torch.sqrt(torch.where(pos, d2, torch.ones_like(d2)))
    if family == ref.MATERN12:
        kap = torch.exp(-d)
    elif family == ref.MATERN32:
        kap = (1.0 + math.sqrt(3.0) * d) * torch.exp(-math.sqrt(3.0) * d)
    else:
        s5 = math.sqrt(5.0) * d
        kap = (1.0 + s5 + s5 * s5 / 3.0) * torch.exp(-s5)
    return var * torch.where(pos, kap, torch.ones_like(kap))


def torch_objective(torch, family, var, t, c, X, Z, y, s, m, jit, objective):
    """log N(y | m, Qxx + S) - [objective == elbo] 1/2 tr(S^-1 (Kxx - Qxx)), Qxx = K_xz (K_zz + J)^-1 K_zx"""
    N, M = X.shape[0], Z.shape[0]
    Kzz = _torch_kernel(torch, family, var, t, c, Z, Z, True) + jit * torch.eye(M, dtype=torch.float64)
    Kxz = _torch_kernel(torch, family, var, t, c, X, Z, False)
    Lz = torch.linalg.cholesky(Kzz)
    P = torch.linalg.solve_triangular(Lz, Kxz.T, upper=False)
    Q = P.T @ P
    Sy = torch.diag(s * torch.ones(N, dtype=torch.float64)) if s.dim() == 0 else torch.diag(s)
    L = torch.linalg.cholesky(Q + Sy)
    r = torch.as_tensor(y) - m
    w = torch.linalg.solve_triangular(L, r[:, None], upper=False)
    f = -0.5 * (N * math.log(2 * math.pi) + 2.0 * torch.log(torch.diagonal(L)).sum() + (w * w).sum())
    if objective == 0:
        kd = torch.diagonal(_torch_kernel(torch, family, var, t, c, X, X, True))
        sv = s * torch.ones(N, dtype=torch.float64) if s.dim() == 0 else s
        f = f - 0.5 * ((kd - torch.diagonal(Q)) / sv).sum()
    return f


def torch_grad(k, mean, noise, X, y, Z, jitter, objective):
    torch = pytest.importorskip("torch")
    N, D = X.shape
    T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), dtype=torch.float64, requires_grad=True)  # noqa: E731
    var = T(k.variance)
    sc = T(k.scale)
    ard = T(k.ard if k.ard is not None else np.ones(D))
    lc = T(k.linear_c)
    t = sc * torch.ones(D, dtype=torch.float64) if k.transform == ref.T_SCALE else (
        ard if k.transform == ref.T_ARD else torch.ones(D, dtype=torch.float64))
    s = T(noise.s if noise.kind == 0 else noise.v)
    mc = T(mean.c)
    mv = T(mean.v if mean.kind == 2 else np.zeros(N))
    m = mc * torch.ones(N, dtype=torch.float64) if mean.kind == 1 else (mv if mean.kind == 2 else torch.zeros(N, dtype=torch.float64))
    Zt = T(Z)
    f = torch_objective(torch, k.family, var, t, lc, torch.as_tensor(X), Zt, y, s, m, jitter.s, objective)
    f.backward()
    g = {"variance": var.grad.item(), "noise": s.grad.item() if noise.kind == 0 else s.grad.numpy()}
    if k.transform == ref.T_SCALE:
        g["scale"] = sc.grad.item()
    elif k.transform == ref.T_ARD:
        g["ard"] = ard.grad.numpy()
    if k.family == ref.LINEAR:
        g["linear_c"] = lc.grad.item()
    if mean.kind == 1:
        g["mean_c"] = mc.grad.item()
    elif mean.kind == 2:
        g["mean_v"] = mv.grad.numpy()
    return f.item(), g, Zt.grad.numpy()


# ---- problems ---------------------------------------------------------------------------------------------------------
def problem(family, transform, noise_kind, mean_kind, N=57, M=11, D=3, seed=0, coincident=False):
    rng = np.random.default_rng(seed + 7 * family + 31 * transform + 101 * noise_kind + 401 * mean_kind + N + M)
    ard = rng.uniform(0.6, 1.4, D) if transform == ref.T_ARD else None
    k = ref.KernelSpec(family, 1.3, transform, scale=0.8, ard=ard, linear_c=0.4 if family == ref.LINEAR else 0.0)
    X = rng.uniform(-2, 2, (N, D))
    Z = rng.uniform(-2, 2, (M, D))
    if coincident:
        Z[1] = X[3]
        Z[4] = X[N - 2]
    y = np.sin(1.5 * X).sum(1) + 0.2 * rng.normal(size=N)
    noise = ref.NoiseSpec(0, 0.15) if noise_kind == 0 else ref.NoiseSpec(1, v=rng.uniform(0.05, 0.3, N))
    mean = [ref.MeanSpec(), ref.MeanSpec(1, 0.3), ref.MeanSpec(2, v=0.2 * rng.normal(size=N))][mean_kind]
    # Linear: K_zz has rank D + 1, so M > D + 1 inducing points need a real jitter
    jitter = ref.NoiseSpec(0, 1e-1 if family == ref.LINEAR else 1e-6)
    return k, mean, noise, X, y, Z, jitter


def assert_grad_close(g, gt, rtol, label=""):
    assert g.keys() == gt.keys(), (label, g.keys(), gt.keys())
    for key in g:
        a, b = np.atleast_1d(g[key]), np.atleast_1d(gt[key])
        np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * max(1.0, np.abs(b).max()), err_msg="%s %s" % (label, key))


MATRIX = list(itertools.product(FAMILIES, [ref.T_NONE, ref.T_SCALE, ref.T_ARD], [0, 1], [0, 1, 2], [0, 1]))


@pytest.mark.parametrize("family,transform,noise_kind,mean_kind,objective", MATRIX)
def test_model_matches_torch_autograd(family, transform, noise_kind, mean_kind, objective):
    # coincident z / x points on every other case, and M > N on every fifth
    idx = MATRIX.index((family, transform, noise_kind, mean_kind, objective))
    N, M = (9, 14) if idx % 5 == 0 and family != ref.LINEAR else (57, 11)
    k, mean, noise, X, y, Z, jitter = problem(family, transform, noise_kind, mean_kind, N=N, M=M, coincident=idx % 2 == 0)
    v, g, z = vg.vfe_grad(k, mean, noise, X, y, Z, jitter, objective)
    vt, gt, zt = torch_grad(k, mean, noise, X, y, Z, jitter, objective)
    assert abs(v - vt) <= 1e-10 * max(1.0, abs(vt))
    assert_grad_close(g, gt, 1e-10)
    np.testing.assert_allclose(z, zt, rtol=1e-10, atol=1e-10 * max(1.0, np.abs(zt).max()))


def test_model_covers_the_linear_kdiag_term():
    """Linear kdiag = sigma_f^2 (||x~||^2 + c) depends on every hyper-parameter: the elbo's variance, scale and c
    derivatives differ from the DTC ones by exactly the kdiag term"""
    k, mean, noise, X, y, Z, jitter = problem(ref.LINEAR, ref.T_SCALE, 0, 1)
    _, ge, _ = vg.vfe_grad(k, mean, noise, X, y, Z, jitter, 0)
    _, gd, _ = vg.vfe_grad(k, mean, noise, X, y, Z, jitter, 1)
    gkd = vg._kdiag_grad(k, X, -np.full(X.shape[0], 0.5 / noise.s))
    assert abs(gkd["scale"]) > 1e-3 and abs(gkd["linear_c"]) > 1e-3
    _, gt, _ = torch_grad(k, mean, noise, X, y, Z, jitter, 0)
    assert_grad_close(ge, gt, 1e-10)
    assert abs(ge["scale"] - gd["scale"]) > 1e-3


@pytest.mark.parametrize("objective", [0, 1])
@pytest.mark.parametrize("case", [(ref.SE, ref.T_ARD, 1, 1), (ref.MATERN52, ref.T_SCALE, 0, 2), (ref.LINEAR, ref.T_ARD, 1, 0)])
def test_model_matches_central_differences(case, objective):
    family, transform, nk, mk = case
    k, mean, noise, X, y, Z, jitter = problem(family, transform, nk, mk, N=40, M=8)
    f = ref.elbo if objective == 0 else ref.dtc
    v, g, z = vg.vfe_grad(k, mean, noise, X, y, Z, jitter, objective)
    h = 1e-6
    for (i, d) in [(0, 0), (3, 2), (7, 1)]:
        Zp, Zm = Z.copy(), Z.copy()
        Zp[i, d] += h
        Zm[i, d] -= h
        fd = (f(k, mean, noise, X, y, Zp, jitter) - f(k, mean, noise, X, y, Zm, jitter)) / (2 * h)
        assert abs(z[i, d] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, d, z[i, d], fd)
    kp, km = ref.KernelSpec(**{**k.__dict__, "variance": k.variance + h}), ref.KernelSpec(**{**k.__dict__, "variance": k.variance - h})
    fd = (f(kp, mean, noise, X, y, Z, jitter) - f(km, mean, noise, X, y, Z, jitter)) / (2 * h)
    assert abs(g["variance"] - fd) <= 1e-6 * max(1.0, abs(fd))


@pytest.mark.parametrize("objective", [0, 1])
@pytest.mark.parametrize("family", FAMILIES)
def test_model_value_is_the_oracle_objective(family, objective):
    k, mean, noise, X, y, Z, jitter = problem(family, ref.T_ARD, 1, 2)
    v, _, _ = vg.vfe_grad(k, mean, noise, X, y, Z, jitter, objective)
    want = (ref.elbo if objective == 0 else ref.dtc)(k, mean, noise, X, y, Z, jitter)
    assert abs(v - want) <= 1e-12 * max(1.0, abs(want))


# ---- the Python mirror through a stand-in library ---------------------------------------------------------------------
class VfeGradFakeLib(fake_libagp.FakeLib):
    """answers agp_vfe_elbo_grad from the model and records its arguments"""

    def __init__(self):
        super().__init__()
        self.calls = []

    def agp_vfe_elbo_grad(self, ctx, dtype, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, objective, value_out,
                          grad_out, noise_diag_out, mean_diag_out, z_grad_out):
        if objective not in (0, 1) or layout not in (0, 1):
            return self._fail(fake_libagp.INVALID, "bad objective or layout")
        dt, ks, ms, ns, Xa, Za, js, ya = self._vfe(dtype, k, mean, noise, layout, X, N, D, Zind, M, jitter, y)
        Xa, Za, ya = Xa.astype(np.float64), Za.astype(np.float64), ya.astype(np.float64)
        v, g, z = vg.vfe_grad(ks, ms, ns, Xa, ya, Za, js, objective)
        self.calls.append({"objective": objective, "layout": layout, "nd": bool(noise_diag_out), "md": bool(mean_diag_out),
                           "z": bool(z_grad_out)})
        fake_libagp._arr(value_out, (1,), dt)[0] = v
        ga = np.ctypeslib.as_array(grad_out, shape=(5 + D,))
        ga[:] = 0.0
        ga[0] = g["variance"]
        ga[1] = g.get("scale", 0.0)
        ga[2] = g.get("linear_c", 0.0)
        ga[3] = np.sum(g["noise"])
        if "ard" in g:
            ga[5:] = g["ard"]
        sbar, mbar = self._per_point(ks, ms, ns, Xa, ya, Za, js, objective)
        ga[4] = np.sum(mbar)
        if noise_diag_out:
            fake_libagp._arr(noise_diag_out, (N,), dt)[:] = sbar
        if mean_diag_out:
            fake_libagp._arr(mean_diag_out, (N,), dt)[:] = mbar
        if z_grad_out:
            out = fake_libagp._arr(z_grad_out, (D, M) if layout == 0 else (M, D), dt, "F")
            out[...] = z.T if layout == 0 else z
        return 0

    @staticmethod
    def _per_point(ks, ms, ns, X, y, Z, js, objective):
        _, g1, _ = vg.vfe_grad(ks, ms, ref.NoiseSpec(1, v=ns.diag(len(y), np.float64)), X, y, Z, js, objective)
        _, g2, _ = vg.vfe_grad(ks, ref.MeanSpec(2, v=ms.vector(len(y), np.float64)), ns, X, y, Z, js, objective)
        return g1["noise"], g2["mean_v"]


@pytest.fixture
def fake(ag, monkeypatch):
    eng = ag.api.Engine.__new__(ag.api.Engine)
    eng.L, eng.h, eng.device = VfeGradFakeLib(), C.c_void_p(1), 0
    monkeypatch.setattr(ag.api, "_engine", eng)
    return eng


def _ag_problem(ag, container, dtype, per_point, mean_kind):
    rng = np.random.default_rng(3)
    D = 1 if container == "vec" else 2
    X = rng.uniform(-2, 2, (30, D)).astype(dtype)
    Z = rng.uniform(-2, 2, (6, D)).astype(dtype)
    y = np.sin(X).sum(1).astype(dtype)
    wrap = {"row": lambda A: ag.RowVecs(A), "col": lambda A: ag.ColVecs(A.T.copy()), "vec": lambda A: A[:, 0].copy()}[container]
    k = 1.2 * ag.with_lengthscale(ag.SqExponentialKernel(), 0.9)
    mean = {0: None, 1: 0.3, 2: (lambda x: 0.1)}[mean_kind]
    f = ag.GP(k) if mean is None else ag.GP(mean, k)
    s2 = rng.uniform(0.05, 0.2, 30).astype(dtype) if per_point else 0.1
    return f, f(wrap(X), s2), f(wrap(Z), 1e-6), y, X, Z, D


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("container", ["row", "col", "vec"])
def test_mirror_shapes_keys_and_objective(ag, fake, dtype, container):
    f, fx, fz, y, X, Z, D = _ag_problem(ag, container, dtype, per_point=container == "col", mean_kind=1)
    v, g = ag.elbo_grad(ag.VFE(fz), fx, y)
    call = fake.L.calls[-1]
    assert call["objective"] == 0 and call["z"] and call["nd"] == (container == "col")
    assert set(g) == {"variance", "scale", "noise", "mean_c", "z"}
    shape = {"row": (6, D), "col": (D, 6), "vec": (6,)}[container]
    assert g["z"].shape == shape and g["z"].dtype == dtype
    assert np.ndim(g["noise"]) == (1 if container == "col" else 0)
    want_v, want, want_z = vg.vfe_grad(ref.KernelSpec(ref.SE, 1.2, ref.T_SCALE, scale=1 / 0.9), ref.MeanSpec(1, 0.3),
                                       ref.NoiseSpec(1, v=fx.Sigma_y_diag.astype(np.float64)) if container == "col"
                                       else ref.NoiseSpec(0, 0.1), X.astype(np.float64), y.astype(np.float64),
                                       Z.astype(np.float64), ref.NoiseSpec(0, 1e-6), 0)
    tol = 1e-10 if dtype == np.float64 else 1e-4
    got_z = {"row": lambda: g["z"], "col": lambda: g["z"].T, "vec": lambda: g["z"][:, None]}[container]()
    np.testing.assert_allclose(got_z, want_z, rtol=tol, atol=tol * np.abs(want_z).max())
    assert abs(g["variance"] - want["variance"]) <= tol * max(1.0, abs(want["variance"]))
    assert abs(v - want_v) <= tol * max(1.0, abs(want_v))
    v1, g1 = ag.approx_log_evidence_grad(ag.DTC(fz), fx, y)
    assert fake.L.calls[-1]["objective"] == 1


def test_mirror_vector_mean_and_dtc_rejection(ag, fake):
    f, fx, fz, y, X, Z, D = _ag_problem(ag, "row", np.float64, per_point=False, mean_kind=2)
    v, g = ag.approx_log_evidence_grad(ag.VFE(fz), fx, y)
    assert fake.L.calls[-1]["md"] and g["mean_v"].shape == (30,)
    with pytest.raises(TypeError):
        ag.elbo_grad(ag.DTC(fz), fx, y)


# ---- ptxas ------------------------------------------------------------------------------------------------------------
def test_vfe_grad_kernels_do_not_spill(tmp_path):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "vfe_grad.cu"), "-o", str(tmp_path / "vfe_grad.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    entries, cur = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
            entries[cur] = []
        elif cur is not None:
            entries[cur].append(line)
    names = {"vfe_cross_grad_kernel": 2, "vfe_point_grad_kernel": 1, "vfe_hz_kernel": 1, "vfe_z_finish_kernel": 1,
             "cast_kernel": 2}
    for kname, count in names.items():
        found = [k for k in entries if kname in k]
        assert len(found) == count, (kname, list(entries))
        for name in found:
            frame = [l for l in entries[name] if "stack frame" in l]
            assert frame, name
            assert all("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in l for l in frame), (name, frame)
