"""The gradient of the VFE objectives with respect to the training inputs (agp_vfe_elbo_grad_x) without a GPU: the NumPy
model tests/vfe_grad_x_ref.py pinned against torch fp64 autograd of the dense restatement of both objectives in
tests/test_vfe_grad_model.py (with X requiring grad) and against central differences; the Python mirror driven through a
stand-in library; and ptxas on the new kernels."""
import os
import re
import subprocess

import numpy as np
import pytest

import fake_libagp
import vfe_grad_x_ref as vx
from oracle import agp_ref as ref
from test_vfe_grad_model import MATRIX, NVCC, CSRC, ROOT, VfeGradFakeLib, _ag_problem, problem, torch_objective


def torch_grad_x(k, mean, noise, X, y, Z, jitter, objective):
    torch = pytest.importorskip("torch")
    N, D = X.shape
    t = torch.ones(D, dtype=torch.float64)
    if k.transform == ref.T_SCALE:
        t = k.scale * t
    elif k.transform == ref.T_ARD:
        t = torch.tensor(np.asarray(k.ard, np.float64))
    s = torch.tensor(noise.s if noise.kind == 0 else np.asarray(noise.v, np.float64), dtype=torch.float64)
    m = torch.tensor(mean.vector(N, np.float64))
    Xt = torch.tensor(np.asarray(X, np.float64), requires_grad=True)
    f = torch_objective(torch, k.family, k.variance, t, k.linear_c, Xt, torch.tensor(np.asarray(Z, np.float64)), y, s, m,
                        jitter.s, objective)
    f.backward()
    return Xt.grad.numpy()


@pytest.mark.parametrize("family,transform,noise_kind,mean_kind,objective", MATRIX)
def test_model_matches_torch_autograd(family, transform, noise_kind, mean_kind, objective):
    # coincident z / x points (Z[1] = X[3], Z[4] = X[N - 2]) on every other case, and M > N on every fifth
    idx = MATRIX.index((family, transform, noise_kind, mean_kind, objective))
    N, M = (9, 14) if idx % 5 == 0 and family != ref.LINEAR else (57, 11)
    k, mean, noise, X, y, Z, jitter = problem(family, transform, noise_kind, mean_kind, N=N, M=M, coincident=idx % 2 == 0)
    x, xs = vx.vfe_grad_x(k, mean, noise, X, y, Z, jitter, objective)
    xt = torch_grad_x(k, mean, noise, X, y, Z, jitter, objective)
    assert np.all(np.isfinite(x))
    np.testing.assert_allclose(x, xt, rtol=1e-10, atol=1e-10 * max(1.0, np.abs(xt).max()))
    assert xs >= 0.5 * np.abs(xt).max()


@pytest.mark.parametrize("family", [ref.SE, ref.MATERN12, ref.MATERN52])
def test_coincident_points_contribute_zero(family):
    """x_3 sits on z_1: the pair's term is exactly 0 (the limit, or for Matern 1/2 the zero subgradient), so xbar_3 is
    the sum over the other inducing points alone"""
    k, mean, noise, X, y, Z, jitter = problem(family, ref.T_SCALE, 0, 1, coincident=True)
    x, _ = vx.vfe_grad_x(k, mean, noise, X, y, Z, jitter, 0)
    W = vx.kbar_zx(k, mean, noise, X, y, Z, jitter, 0)
    W[1, 3] = 0.0
    _, cross = vx._contract(k, X, Z, W.T)
    assert np.all(np.isfinite(x))
    np.testing.assert_array_equal(x[3], cross[3])


def test_model_covers_the_linear_kdiag_term():
    """for the Linear kernel the elbo's xbar differs from DTC's by the kdiag term -sigma^2 t^2 x / s (and by c in
    Kbar_zx); torch agrees on both"""
    k, mean, noise, X, y, Z, jitter = problem(ref.LINEAR, ref.T_ARD, 1, 0)
    for objective in (0, 1):
        x, _ = vx.vfe_grad_x(k, mean, noise, X, y, Z, jitter, objective)
        xt = torch_grad_x(k, mean, noise, X, y, Z, jitter, objective)
        np.testing.assert_allclose(x, xt, rtol=1e-10, atol=1e-10 * np.abs(xt).max())
    t = np.asarray(k.ard)
    assert np.abs(k.variance * t * t * X / noise.v[:, None]).max() > 1e-2


def test_translation_invariance_of_the_model():
    """a stationary kernel: shifting every x and z by the same vector leaves the objective unchanged, so
    sum_n xbar_n + sum_m zbar_m = 0"""
    import vfe_grad_ref as vg
    for family in (ref.SE, ref.MATERN32):
        k, mean, noise, X, y, Z, jitter = problem(family, ref.T_ARD, 1, 2)
        x, xs = vx.vfe_grad_x(k, mean, noise, X, y, Z, jitter, 0)
        _, _, z = vg.vfe_grad(k, mean, noise, X, y, Z, jitter, 0)
        np.testing.assert_allclose(x.sum(0) + z.sum(0), 0.0, atol=1e-11 * max(xs, np.abs(z).max()))


@pytest.mark.parametrize("objective", [0, 1])
@pytest.mark.parametrize("case", [(ref.SE, ref.T_ARD, 1, 1), (ref.MATERN52, ref.T_SCALE, 0, 2), (ref.LINEAR, ref.T_ARD, 1, 0),
                                  (ref.MATERN12, ref.T_NONE, 0, 0)])
def test_model_matches_central_differences(case, objective):
    family, transform, nk, mk = case
    k, mean, noise, X, y, Z, jitter = problem(family, transform, nk, mk, N=40, M=8)
    f = ref.elbo if objective == 0 else ref.dtc
    x, _ = vx.vfe_grad_x(k, mean, noise, X, y, Z, jitter, objective)
    h = 1e-6
    for (i, d) in [(0, 0), (3, 2), (17, 1), (39, 0)]:
        Xp, Xm = X.copy(), X.copy()
        Xp[i, d] += h
        Xm[i, d] -= h
        fd = (f(k, mean, noise, Xp, y, Z, jitter) - f(k, mean, noise, Xm, y, Z, jitter)) / (2 * h)
        assert abs(x[i, d] - fd) <= 1e-6 * max(1.0, abs(fd)), (i, d, x[i, d], fd)


# ---- the Python mirror through a stand-in library ---------------------------------------------------------------------
class VfeGradXFakeLib(VfeGradFakeLib):
    """VfeGradFakeLib plus agp_vfe_elbo_grad_x; every call records the symbol it came through"""

    def agp_vfe_elbo_grad(self, *args):
        rc = super().agp_vfe_elbo_grad(*args)
        if rc == 0:
            self.calls[-1]["symbol"] = "agp_vfe_elbo_grad"
        return rc

    def agp_vfe_elbo_grad_x(self, ctx, dtype, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, objective, value_out,
                            grad_out, noise_diag_out, mean_diag_out, z_grad_out, x_grad_out):
        rc = super().agp_vfe_elbo_grad(ctx, dtype, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, objective,
                                       value_out, grad_out, noise_diag_out, mean_diag_out, z_grad_out)
        if rc:
            return rc
        dt, ks, ms, ns, Xa, Za, js, ya = self._vfe(dtype, k, mean, noise, layout, X, N, D, Zind, M, jitter, y)
        x, _ = vx.vfe_grad_x(ks, ms, ns, Xa.astype(np.float64), ya.astype(np.float64), Za.astype(np.float64), js, objective)
        self.calls[-1].update(symbol="agp_vfe_elbo_grad_x", x=bool(x_grad_out))
        if x_grad_out:
            out = fake_libagp._arr(x_grad_out, (D, N) if layout == 0 else (N, D), dt, "F")
            out[...] = x.T if layout == 0 else x
        return 0


@pytest.fixture
def fake(ag, monkeypatch):
    import ctypes as C
    eng = ag.api.Engine.__new__(ag.api.Engine)
    eng.L, eng.h, eng.device = VfeGradXFakeLib(), C.c_void_p(1), 0
    monkeypatch.setattr(ag.api, "_engine", eng)
    return eng


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("container", ["row", "col", "vec"])
def test_mirror_inputs_shapes_and_symbol(ag, fake, dtype, container):
    f, fx, fz, y, X, Z, D = _ag_problem(ag, container, dtype, per_point=container == "col", mean_kind=2)
    n0 = len(fake.L.calls)
    v0, g0 = ag.elbo_grad(ag.VFE(fz), fx, y)
    assert len(fake.L.calls) == n0 + 1 and fake.L.calls[-1]["symbol"] == "agp_vfe_elbo_grad" and "x" not in g0
    v, g = ag.elbo_grad(ag.VFE(fz), fx, y, inputs=True)
    assert len(fake.L.calls) == n0 + 2
    call = fake.L.calls[-1]
    assert call["symbol"] == "agp_vfe_elbo_grad_x" and call["x"] and call["objective"] == 0
    assert set(g) == set(g0) | {"x"}
    shape = {"row": (30, D), "col": (D, 30), "vec": (30,)}[container]
    assert g["x"].shape == shape and g["x"].dtype == dtype
    for key in g0:
        np.testing.assert_array_equal(np.asarray(g[key]), np.asarray(g0[key]), err_msg=key)
    want, _ = vx.vfe_grad_x(ref.KernelSpec(ref.SE, 1.2, ref.T_SCALE, scale=1 / 0.9),
                            ref.MeanSpec(2, v=np.full(30, 0.1)),
                            ref.NoiseSpec(1, v=fx.Sigma_y_diag.astype(np.float64)) if container == "col"
                            else ref.NoiseSpec(0, 0.1), X.astype(np.float64), y.astype(np.float64),
                            Z.astype(np.float64), ref.NoiseSpec(0, 1e-6), 0)
    got = {"row": lambda: g["x"], "col": lambda: g["x"].T, "vec": lambda: g["x"][:, None]}[container]()
    tol = 1e-10 if dtype == np.float64 else 1e-4
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol * np.abs(want).max())
    v1, g1 = ag.approx_log_evidence_grad(ag.DTC(fz), fx, y, inputs=True)
    assert fake.L.calls[-1]["symbol"] == "agp_vfe_elbo_grad_x" and fake.L.calls[-1]["objective"] == 1
    assert g1["x"].shape == shape


# ---- ptxas ------------------------------------------------------------------------------------------------------------
def test_vfe_grad_x_kernels_do_not_spill(tmp_path):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "vfe_grad_x.cu"), "-o", str(tmp_path / "vfe_grad_x.o")]
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
    assert len(entries) == 3, list(entries)
    for kname, count in {"vfe_x_grad_kernel": 2, "vfe_x_finish_kernel": 1}.items():
        found = [k for k in entries if kname in k]
        assert len(found) == count, (kname, list(entries))
        for name in found:
            frame = [l for l in entries[name] if "stack frame" in l]
            assert frame, name
            assert all("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in l for l in frame), (name, frame)
