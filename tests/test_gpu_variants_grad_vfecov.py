"""Variants of the int8-slice trailing-update kernel, the device gradient of logpdf, the full covariance of the approximate
posterior and the replays of the reference's own test sets.  The kernel variants run in subprocesses under a timeout, so a
protocol bug (the mbarrier spin limit traps) fails one test instead of poisoning the session.  Each must be bit-identical
to the default launch (persistent grid, int32 pair pre-combination in the drain where K <= 512):

* AGP_OZAKI_EPI=0 -- the plain int64 drain (the same exact integers, so the same single rounding);
* AGP_OZAKI_CHUNK_TEST=1 / =4 -- bounded CTAs of 1 / 4 consecutive tiles each (the form the look-ahead schedule uses)
  instead of the persistent grid of the debug entry."""
import os
import subprocess
import sys

import pytest

pytestmark = [pytest.mark.gpu]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("switches", [["AGP_OZAKI_EPI=0"], ["AGP_OZAKI_CHUNK_TEST=1"],
                                      ["AGP_OZAKI_EPI=0", "AGP_OZAKI_CHUNK_TEST=4"], ["AGP_OZAKI_CHUNK_TEST=4"]])
@pytest.mark.parametrize("N,K,S", [(128, 128, 7), (1024, 256, 7), (4224, 512, 7), (2176, 512, 6), (8192, 512, 7), (1152, 1024, 8)])
def test_variant_matches_default_kernel(N, K, S, switches):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "exp_variant_check.py"), str(N), str(K), str(S)] + switches,
                       capture_output=True, text=True, timeout=180, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    line = [l for l in r.stdout.splitlines() if l.startswith("MAXDIFF")][-1].split()
    assert float(line[1]) == 0.0, line
    assert float(line[3]) > 0.0, line  # the update really happened


# ---- SURVEY s8(f) rank 1: gradient of logpdf on the device (agp_post_logpdf_grad, csrc/grad.cu) vs the gradient oracle
@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
@pytest.mark.parametrize("transform", ["scale", "ard"])
@pytest.mark.parametrize("fam", [0, 1, 2, 3, 4])
def test_logpdf_grad_matches_oracle(ag, fam, transform, dtype_name):
    import numpy as np
    from oracle import agp_ref as ref
    from test_gpu_parity import FAM_CTOR
    dtype = np.dtype(dtype_name).type
    rng = np.random.default_rng(5)
    n, D = 333, 5
    X = rng.random((n, D)).astype(dtype)
    y = (np.sin(3 * X[:, 0]) + 0.2 * rng.standard_normal(n)).astype(dtype)
    ard = (0.6 + rng.random(D)).astype(dtype)
    ks = ref.KernelSpec(fam, 1.3, ref.T_SCALE if transform == "scale" else ref.T_ARD, scale=1.7, ard=ard, linear_c=0.4)
    nv = (0.05 + 0.1 * rng.random(n)).astype(dtype)
    k = getattr(ag, FAM_CTOR[fam])() if fam != ref.LINEAR else ag.LinearKernel(c=0.4)
    k = 1.3 * k.compose(ag.ScaleTransform(1.7) if transform == "scale" else ag.ARDTransform(ard))
    f = ag.GP(0.25, k)
    lp, g = ag.logpdf_grad(f(ag.RowVecs(X), nv), y)
    want = ref.logpdf_grad(ks, ref.MeanSpec(1, 0.25), ref.NoiseSpec(1, v=nv), X.astype(np.float64), y.astype(np.float64))
    rt = 1e-7 if dtype == np.float64 else 2e-2
    scale_of = lambda a: max(1.0, float(np.max(np.abs(a))))
    for key in ("variance", "mean_c", "noise") + (("scale",) if transform == "scale" else ("ard",)) + (("linear_c",) if fam == 4 else ()):
        np.testing.assert_allclose(g[key], want[key], rtol=rt, atol=rt * scale_of(want[key]), err_msg=key)
    assert np.isclose(lp, ref.logpdf(ks, ref.MeanSpec(1, 0.25), ref.NoiseSpec(1, v=nv), X, y), rtol=1e-8 if dtype == np.float64 else 1e-4)


# ---- the reference's own test sets for the hot path (tests/ref_suite_replays.py) on the device; their logic already
# runs on the CPU against the fake library (tests/test_api_on_fake_lib.py) -- promote to the default GPU suite once green
def test_reference_finite_gp_testsets_on_device(ag):
    import numpy as np
    import ref_suite_replays as rs
    rs.finite_gp_statistics(ag)
    rs.finite_gp_rand_statistical(ag)
    rs.finite_gp_logpdf(ag)
    for T in (np.float64, np.float32):
        rs.finite_gp_type_stability(ag, T)


@pytest.mark.parametrize("approx_name", ["VFE", "DTC"])
def test_reference_sparse_testsets_on_device(ag, approx_name):
    import numpy as np
    import ref_suite_replays as rs
    A = getattr(ag, approx_name)
    rs.sparse_approx_log_evidence(ag, A)
    rs.sparse_posterior_matches_exact(ag, A)
    rs.sparse_update_posterior(ag, A)
    import test_gpu_posterior_finitegp as pf
    rs.sparse_internal_interface(ag, A, pf)
    for T in (np.float64, np.float32):
        rs.sparse_type_stability(ag, A, T)


@pytest.mark.parametrize("dtype_name", ["float64", "float32"])
def test_vfe_cov_logpdf_rand_match_oracle(ag, dtype_name):
    """agp_vfe_mean_cov / agp_vfe_post_logpdf / agp_vfe_post_rand (full covariance of the approximate posterior and a
    FiniteGP over it) against the oracle."""
    import numpy as np
    from oracle import agp_ref as ref
    dtype = np.dtype(dtype_name).type
    rng = np.random.default_rng(8)
    n, m, d, M = 900, 140, 3, 200
    X, Zi, Xs = rng.random((n, d)).astype(dtype), rng.random((m, d)).astype(dtype), rng.random((M, d)).astype(dtype)
    y = (np.sin(3 * X[:, 0]) + 0.1 * rng.standard_normal(n)).astype(dtype)
    ks = ref.KernelSpec(ref.MATERN52, 1.2, ref.T_SCALE, scale=2.0)
    f = ag.GP(0.2, 1.2 * ag.Matern52Kernel().compose(ag.ScaleTransform(2.0)))
    jit = 1e-6 if dtype == np.float64 else 1e-4
    post = ag.posterior(ag.VFE(f(ag.RowVecs(Zi), jit)), f(ag.RowVecs(X), 0.1), y)
    vp = ref.vfe_posterior(ks, ref.MeanSpec(1, 0.2), ref.NoiseSpec(0, 0.1), X, y, Zi, ref.NoiseSpec(0, jit))
    mr, Cr = ref.vfe_mean_and_cov(vp, Xs)
    m_, C_ = ag.mean_and_cov(post, ag.RowVecs(Xs))
    tol = dict(rtol=1e-6, atol=1e-7) if dtype == np.float64 else dict(rtol=2e-2, atol=2e-3)
    assert np.allclose(m_, mr, **tol) and np.allclose(C_, Cr, **tol)
    assert np.allclose(ag.cov(post, ag.RowVecs(Xs[:50]), ag.RowVecs(Xs[50:90])), ref.vfe_cov_cross(vp, Xs[:50], Xs[50:90]), **tol)
    Cn = Cr.astype(np.float64) + 0.05 * np.eye(M)
    U = ref.cholesky_upper(Cn)
    Ys = rng.standard_normal((M, 2)).astype(dtype)
    want = -0.5 * (M * ref.LOG2PI + ref.logdet_chol(U) + ref.diag_Xt_invA_X(U, Ys.astype(np.float64) - mr[:, None]))
    got = ag.logpdf(post(ag.RowVecs(Xs), 0.05), Ys)
    assert np.allclose(got, want, rtol=1e-8 if dtype == np.float64 else 2e-3)
    Zn = rng.standard_normal((M, 3)).astype(dtype)
    got_r = ag.rand_from_normals(post(ag.RowVecs(Xs), 0.05), Zn)
    assert np.allclose(got_r, mr[:, None] + U.T @ Zn, **(dict(rtol=0, atol=1e-7) if dtype == np.float64 else dict(rtol=0, atol=5e-3)))
