"""The oracle's VFE objective pinned at the size where the GPU cases of tests/test_gpu_vfe_tensor.py live (N = 3000,
M = 1100, the C5 kernel).  tests/test_oracle_independent_pins.py checks `elbo` / `dtc` against 60-digit arithmetic at
N = 12, M = 5 only; at M = 1100 cond(K_zz + jitter) is ~2e7, and a 1e-8 comparison of a CUDA result with the oracle is
worth no more than the oracle's own digits there.

The second formulation is the textbook dense one (Titsias 2009, eq. 9),
    elbo = log N(y; m, Q + Sigma) - 1/2 tr((K_ff - Q) Sigma^-1),   Q = K_xz (K_zz + J)^-1 K_zx,
on the N x N matrices: Q from an eigendecomposition of K_zz + J, log det(Q + Sigma) from its eigenvalues, the quadratic
form from a symmetric-positive solve.  It shares the three kernel matrices with `_compute_intermediates`
(the reference's src/sparse_approximations.jl:289-305), which are pinned to scikit-learn on their own, and nothing after
them: no Cholesky factor of K_zz, no A = U' \\ K_zx, no M x M matrix A A' + I, no matrix-determinant lemma.
Measured agreement: 1e-14 .. 7e-14 relative for jitter 1e-8, 1e-6 and 1e-4, so the GPU cases may ask for 1e-8."""
import numpy as np
import pytest
import scipy.linalg as sla

from oracle import agp_ref as ref


def dense_elbo_dtc(k, mean, noise, X, y, Z, jitter):
    n, M = X.shape[0], Z.shape[0]
    Kzz = ref.kernelmatrix(k, Z)
    Kzz[np.diag_indices(M)] += jitter.diag(M, X.dtype)
    w, V = np.linalg.eigh(Kzz)
    P = ref.kernelmatrix(k, X, Z) @ V
    Q = (P / w) @ P.T
    Q = 0.5 * (Q + Q.T)
    s = noise.diag(n, X.dtype)
    C = Q.copy()
    C[np.diag_indices(n)] += s
    d = y - mean.vector(n, X.dtype)
    logdet = np.sum(np.log(np.linalg.eigvalsh(C)))
    quad = d @ sla.solve(C, d, assume_a="pos")
    dtc = -0.5 * (n * ref.LOG2PI + logdet + quad)
    return dtc - 0.5 * np.sum((np.diag(ref.kernelmatrix(k, X)) - np.diag(Q)) / s), dtc


@pytest.mark.parametrize("jit", [1e-6, 1e-4])
@pytest.mark.parametrize("variant", ["plain", "noise_vector_const_mean"])
def test_vfe_objective_matches_dense_form_at_m1100(jit, variant):
    n, m = 3000, 1100
    cfg = ref.make_config("C5", n=n, dtype=np.float64)
    X, y = cfg["X"], cfg["y"]
    Z = X[np.random.default_rng(7).permutation(n)[:m]].copy()
    mean, noise = cfg["mean"], cfg["noise"]
    if variant != "plain":
        mean = ref.MeanSpec(1, 0.3)
        noise = ref.NoiseSpec(1, v=0.05 + 0.1 * np.random.default_rng(8).random(n))
    jn = ref.NoiseSpec(0, jit)
    el = ref.elbo(cfg["k"], mean, noise, X, y, Z, jn)
    dt = ref.dtc(cfg["k"], mean, noise, X, y, Z, jn)
    el_d, dt_d = dense_elbo_dtc(cfg["k"], mean, noise, X, y, Z, jn)
    assert abs(el - el_d) <= 1e-10 * abs(el_d), (el, el_d)
    assert abs(dt - dt_d) <= 1e-10 * abs(dt_d), (dt, dt_d)
    assert el < dt  # the trace term is a penalty: K_ff - Q is positive semi-definite
