"""CPU model of the gradient of the VFE objectives (agp.h agp_vfe_elbo_grad) in NumPy, fp64, for the single kernels the
VFE path accepts (oracle.agp_ref.KernelSpec).  Test infrastructure only.

Notation (agp.h): Q = K_zz + J = L_z L_z', s_i = sigma_i^2, delta = s^-1/2 (y - m), A = L_z^-1 K_zx S^-1/2,
Lam = I + A A' = L_m L_m', b = A delta, m_e = Lam^-1 b, c = 1 for the elbo and 0 for DTC.

  F = -1/2 [N log 2pi + sum log s_i + log|Lam| + delta'delta - b' Lam^-1 b] - c/2 [sum kdiag_i / s_i - ||A||_F^2]

With V_z = L_z^-1, H = c I - Lam^-1 - m_e m_e', R = V_z' H V_z, r = V_z' m_e and E = c (Lam - I) - I + Lam^-1 + m_e m_e':
  Kbar_zx = R K_zx S^-1 + r (delta o s^-1/2)'        Kbar_zz = -1/2 V_z' E V_z        kdiagbar_i = -c / (2 s_i)
  u = K_zx' r,  q_i = sum_m Kbar_zx[m, i] K_zx[m, i]
  deltabar = -delta + s^-1/2 u,  sbar = -1/(2s) + c kdiag/(2s^2) - q/(2s) - deltabar delta/(2s),  mbar = -s^-1/2 deltabar
  dF/dtheta = sum Kbar_zz o dK_zz + sum Kbar_zx o dK_zx + sum kdiagbar o dkdiag
  zbar_m = 2 sum_m' Kbar_zz[m, m'] d1k(z_m, z_m') + sum_n Kbar_zx[m, n] d1k(z_m, x_n)"""
import math

import numpy as np
import scipy.linalg as sla

from oracle import agp_ref as ref


def _t(k, D):
    if k.transform == ref.T_SCALE:
        return np.full(D, float(k.scale))
    if k.transform == ref.T_ARD:
        return np.asarray(k.ard, dtype=np.float64)
    return np.ones(D)


def _contract(k, A, B, W, block=None):
    """sum_ab W_ab dK(a, b)/dtheta for every hyper-parameter (dict) and sum_b W_ab d1k(a, b) ((|A|, D), with respect to
    the untransformed a), over blocks of B"""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    D = A.shape[1]
    t = _t(k, D)
    At = A * t
    g = {"variance": 0.0, "scale": 0.0, "linear_c": 0.0, "ard": np.zeros(D)}
    d1 = np.zeros(A.shape)
    block = block or max(1, int(4e6 // max(1, A.shape[0] * D)))
    for j0 in range(0, B.shape[0], block):
        Bj, Wj = B[j0:j0 + block], W[:, j0:j0 + block]
        Bt = Bj * t
        if k.family == ref.LINEAR:
            G = At @ Bt.T
            g["variance"] += np.sum(Wj * (G + k.linear_c))
            g["linear_c"] += k.variance * np.sum(Wj)
            g["scale"] += 2.0 * k.variance * np.sum(Wj * G) / t[0]
            g["ard"] += 2.0 * k.variance * t * np.einsum("ab,ad,bd->d", Wj, A, Bj)
            d1 += k.variance * (Wj @ Bj) * t * t
        else:
            raw = A[:, None, :] - Bj[None, :, :]
            diff = raw * t
            d2 = np.einsum("abd,abd->ab", diff, diff)
            g["variance"] += np.sum(Wj * ref._kappa(k.family, d2))
            KR = k.variance * ref._dkappa_r(k.family, d2)  # sigma_f^2 kappa'(r) r
            g["scale"] += np.sum(Wj * KR) / t[0]
            with np.errstate(divide="ignore", invalid="ignore"):
                Qm = np.where(d2 > 0, KR / np.where(d2 > 0, d2, 1.0), 0.0)  # 2 sigma_f^2 dkappa/dd2, 0 at coincident points
            WQ = Wj * Qm
            g["ard"] += t * np.einsum("ab,abd->d", WQ, raw * raw)
            d1 += np.einsum("ab,abd->ad", WQ, raw) * t * t
    return g, d1


def _kdiag_grad(k, X, w):
    """sum_i w_i dkdiag_i/dtheta"""
    g = {"variance": 0.0, "scale": 0.0, "linear_c": 0.0, "ard": np.zeros(X.shape[1])}
    if k.family != ref.LINEAR:
        g["variance"] = float(np.sum(w))
        return g
    t = _t(k, X.shape[1])
    Xt = X * t
    n2 = np.sum(Xt * Xt, 1)
    g["variance"] = float(np.sum(w * (n2 + k.linear_c)))
    g["linear_c"] = k.variance * float(np.sum(w))
    g["scale"] = 2.0 * k.variance * float(np.sum(w * n2)) / t[0]
    g["ard"] = 2.0 * k.variance * t * np.einsum("i,id->d", w, X * X)
    return g


def vfe_grad(k, mean, noise, X, y, Z, jitter, objective=0, z_scale=False):
    """(value, gradient dict, zbar (M, D)) of the elbo (objective 0) or the DTC objective (1); z_scale=True adds the
    largest entry of the two terms zbar sums (K_zz and K_zx parts), the scale its rounding error is relative to.  The dict has the keys of
    oracle.agp_ref.logpdf_grad for the kernel ("variance", "scale" | "ard", "linear_c"), "noise" (scalar, or the
    per-point vector when noise.kind == 1), and "mean_c" (mean.kind == 1) or "mean_v" (mean.kind == 2)."""
    X, Z = np.asarray(X, np.float64), np.asarray(Z, np.float64)
    y = np.asarray(y, np.float64)
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
    Lam = np.eye(M) + A @ A.T
    Lm = np.linalg.cholesky(Lam)
    b = A @ delta
    me = sla.cho_solve((Lm, True), b)
    kd = ref.kernelmatrix_diag(k, X)
    value = -0.5 * (N * math.log(2 * math.pi) + np.sum(np.log(s)) + 2.0 * np.sum(np.log(np.diag(Lm)))
                    + delta @ delta - b @ me) - c * 0.5 * (np.sum(kd / s) - np.sum(A * A))

    Vz = sla.solve_triangular(Lz, np.eye(M), lower=True)
    Lami = sla.cho_solve((Lm, True), np.eye(M))
    mm = np.outer(me, me)
    H = c * np.eye(M) - Lami - mm
    R = Vz.T @ H @ Vz
    r = Vz.T @ me
    E = c * (Lam - np.eye(M)) - np.eye(M) + Lami + mm
    Kb_zz = -0.5 * Vz.T @ E @ Vz
    Kb_zx = (R @ Kzx) / s + np.outer(r, delta * isn)
    u = Kzx.T @ r
    q = np.sum(Kb_zx * Kzx, 0)
    dbar = -delta + isn * u
    sbar = -0.5 / s + c * kd / (2 * s * s) - q / (2 * s) - dbar * delta / (2 * s)
    mbar = -isn * dbar

    gzz, d1zz = _contract(k, Z, Z, Kb_zz)
    gzx, d1zx = _contract(k, Z, X, Kb_zx)
    gkd = _kdiag_grad(k, X, -c / (2 * s))
    g = {"variance": gzz["variance"] + gzx["variance"] + gkd["variance"]}
    if k.transform == ref.T_SCALE:
        g["scale"] = gzz["scale"] + gzx["scale"] + gkd["scale"]
    elif k.transform == ref.T_ARD:
        g["ard"] = gzz["ard"] + gzx["ard"] + gkd["ard"]
    if k.family == ref.LINEAR:
        g["linear_c"] = gzz["linear_c"] + gzx["linear_c"] + gkd["linear_c"]
    g["noise"] = float(np.sum(sbar)) if noise.kind == 0 else sbar
    if mean.kind == 1:
        g["mean_c"] = float(np.sum(mbar))
    elif mean.kind == 2:
        g["mean_v"] = mbar
    zbar = 2.0 * d1zz + d1zx
    if z_scale:
        return float(value), g, zbar, max(np.abs(2.0 * d1zz).max(), np.abs(d1zx).max())
    return float(value), g, zbar
