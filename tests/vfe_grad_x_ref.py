"""CPU model of the gradient of the VFE objectives with respect to the training inputs (agp.h agp_vfe_elbo_grad_x) in
NumPy, fp64, for the single kernels the VFE path accepts.  Test infrastructure only.

In the notation of tests/vfe_grad_ref.py, with respect to the untransformed inputs:
  xbar_n = sum_m Kbar_zx[m, n] d1k(x_n, z_m) + kdiagbar_n dkdiag(x_n)/dx_n,   kdiagbar_n = -c / (2 s_n)
d1k the derivative in the first argument.  The kdiag term is 0 for the stationary families and -c sigma^2 t^2 x_n / s_n
for the Linear kernel (kdiag = sigma^2 (||t x||^2 + c)).  The mean and per-point noise are constants of x."""
import numpy as np
import scipy.linalg as sla

from oracle import agp_ref as ref
from vfe_grad_ref import _contract, _t


def kbar_zx(k, mean, noise, X, y, Z, jitter, objective=0):
    """Kbar_zx (M, N) of agp.h, from the same intermediates as vfe_grad_ref.vfe_grad"""
    X, Z, y = np.asarray(X, np.float64), np.asarray(Z, np.float64), np.asarray(y, np.float64)
    N, M = X.shape[0], Z.shape[0]
    c = 1.0 if objective == 0 else 0.0
    s = noise.diag(N, np.float64)
    isn = 1.0 / np.sqrt(s)
    delta = (y - mean.vector(N, np.float64)) * isn
    Kzz = ref.kernelmatrix(k, Z)
    Kzz[np.diag_indices(M)] += jitter.diag(M, np.float64)
    Lz = np.linalg.cholesky(Kzz)
    Kzx = ref.kernelmatrix(k, Z, X)
    A = sla.solve_triangular(Lz, Kzx * isn, lower=True)
    Lm = np.linalg.cholesky(np.eye(M) + A @ A.T)
    me = sla.cho_solve((Lm, True), A @ delta)
    Vz = sla.solve_triangular(Lz, np.eye(M), lower=True)
    H = c * np.eye(M) - sla.cho_solve((Lm, True), np.eye(M)) - np.outer(me, me)
    return (Vz.T @ H @ Vz @ Kzx) / s + np.outer(Vz.T @ me, delta * isn)


def vfe_grad_x(k, mean, noise, X, y, Z, jitter, objective=0):
    """(xbar (N, D), x_scale): x_scale is the larger of the two terms xbar sums (the K_zx part and the kdiag part), the
    scale its rounding error is relative to"""
    X = np.asarray(X, np.float64)
    N, D = X.shape
    c = 1.0 if objective == 0 else 0.0
    W = kbar_zx(k, mean, noise, X, y, Z, jitter, objective)
    _, cross = _contract(k, X, Z, W.T)
    kdiag = np.zeros_like(X)
    if k.family == ref.LINEAR:
        t = _t(k, D)
        kdiag = -c * k.variance * (t * t) * X / noise.diag(N, np.float64)[:, None]
    return cross + kdiag, float(max(np.abs(cross).max(), np.abs(kdiag).max()))
