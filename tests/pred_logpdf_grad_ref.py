"""CPU model of the gradient of the held-out log-likelihood sum_s w_s logpdf(posterior(fx, y)(x*, Sigma*), Y*[:, s])
(agp.h agp_post_pred_logpdf_grad), in NumPy fp64, for single kernels (oracle.agp_ref.KernelSpec) and composites
(tests/composite_ref.Composite).  Test infrastructure only.

With C = K_xx + Sigma_y, alpha = C^-1 (y - m), P = C^-1 K_xs, mu* = m* + K_sx alpha, Sigma = K_ss - K_sx P + Sigma*,
E = Y* - mu* 1' and B = Sigma^-1 E (all by Cholesky solves):
    Sigmabar = 1/2 (B diag(w) B' - (sum w) Sigma^-1),  mubar = B w,  Ybar* = -B diag(w),  beta = P mubar
    Kbar_sx = mubar alpha' - 2 Sigmabar P',  Cbar = P Sigmabar P' - 1/2 (beta alpha' + alpha beta')
    ybar = beta,  mbar = -beta,  mbar* = mubar,  d/d sigma_i^2 = Cbar_ii,  d/d sigma*_m^2 = Sigmabar_mm
    d/d theta = <Cbar, dK_xx> + <Kbar_sx, dK_sx> + <Sigmabar, dK_ss>
    x_i  = 2 sum_j Cbar_ij d1k(x_i, x_j) + sum_m Kbar_sx[m, i] d1k(x_i, x*_m)
    x*_m = 2 sum_m' Sigmabar_mm' d1k(x*_m, x*_m') + sum_i Kbar_sx[m, i] d1k(x*_m, x_i)
The kernel terms are taken as 1/2 <W, dK([x; x*])> with W = [2 Cbar, Kbar_xs; Kbar_sx, 2 Sigmabar], the same sum
written over the stacked points (rand_grad_ref.descriptor_grad)."""
import numpy as np
from scipy.linalg import cho_factor, cho_solve

import composite_ref as cr
import grad_x_ref as gx
import rand_grad_ref as rg
from oracle import agp_ref as ref

LOG2PI = np.log(2.0 * np.pi)


def pred_logpdf_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, Ys, w=None):
    """dict: "lp" (S), "grad" (grad_out: 5 + D for a KernelSpec, the descriptor layout for a Composite), "noise_diag",
    "mean_diag", "y" (N), "x" (N x D), "noise_s_diag", "mean_s_diag" (M), "Ys" (M x S), "xs" (M x D).  mean_s is the
    prior mean at Xs (a MeanSpec of the same kind as mean)."""
    X = np.asarray(X, dtype=np.float64)
    Xs = np.asarray(Xs, dtype=np.float64)
    N, D = X.shape
    M = Xs.shape[0]
    Ys = np.asarray(Ys, dtype=np.float64).reshape(M, -1)
    S = Ys.shape[1]
    w = np.ones(S) if w is None else np.asarray(w, dtype=np.float64)
    kc = gx.as_composite(k)
    Kxx = cr.kernelmatrix(kc, X)
    Kxs = cr.kernelmatrix(kc, X, Xs)
    Kss = cr.kernelmatrix(kc, Xs)
    cf = cho_factor(Kxx + np.diag(noise.diag(N, np.float64)), lower=True)
    alpha = cho_solve(cf, np.asarray(y, dtype=np.float64) - mean.vector(N, np.float64))
    P = cho_solve(cf, Kxs)
    mu = mean_s.vector(M, np.float64) + Kxs.T @ alpha
    Sig = Kss - Kxs.T @ P + np.diag(noise_s.diag(M, np.float64))
    sf = cho_factor(Sig, lower=True)
    E = Ys - mu[:, None]
    B = cho_solve(sf, E)
    Sinv = cho_solve(sf, np.eye(M))
    lp = -0.5 * (M * LOG2PI + 2.0 * np.sum(np.log(np.diag(sf[0]))) + np.sum(E * B, axis=0))
    Sbar = 0.5 * ((B * w) @ B.T - np.sum(w) * Sinv)
    mubar = B @ w
    beta = P @ mubar
    Kbar = np.outer(mubar, alpha) - 2.0 * Sbar @ P.T
    Cbar = P @ Sbar @ P.T - 0.5 * (np.outer(beta, alpha) + np.outer(alpha, beta))
    W = np.block([[2.0 * Cbar, Kbar.T], [Kbar, 2.0 * Sbar]])
    gc = rg.descriptor_grad(k, W, np.vstack([X, Xs]))
    if isinstance(k, cr.Composite):
        g = gc
    else:  # the one-factor descriptor [5] variance, [6..] Scale s | ARD v, then Linear c, back to the single layout
        g = np.zeros(5 + D)
        g[0] = gc[5]
        pos = 6
        if k.transform == ref.T_SCALE:
            g[1] = gc[pos]
            pos += 1
        elif k.transform == ref.T_ARD:
            g[5:] = gc[pos:pos + D]
            pos += D
        if k.family == ref.LINEAR:
            g[2] = gc[pos]
    g[3] = np.trace(Cbar)
    g[4] = np.sum(mubar) - np.sum(beta)
    xg = 2.0 * np.einsum("ij,ijd->id", Cbar, gx.kernel_d1(k, X, X)) + np.einsum("mi,imd->id", Kbar, gx.kernel_d1(k, X, Xs))
    xsg = 2.0 * np.einsum("ij,ijd->id", Sbar, gx.kernel_d1(k, Xs, Xs)) + np.einsum("mi,mid->md", Kbar, gx.kernel_d1(k, Xs, X))
    return {"lp": lp, "grad": g, "noise_diag": np.diag(Cbar).copy(), "mean_diag": -beta, "y": beta, "x": xg,
            "noise_s_diag": np.diag(Sbar).copy(), "mean_s_diag": mubar, "Ys": -B * w, "xs": xsg}
