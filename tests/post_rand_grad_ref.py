"""CPU model of the pullback of rand over an exact posterior, out = mu* 1' + L* Z for posterior(fx, y)(x*, Sigma*)
(agp.h agp_post_rand_grad), in NumPy fp64, for single kernels (oracle.agp_ref.KernelSpec) and composites
(tests/composite_ref.Composite).  Test infrastructure only.

With C = K_xx + Sigma_y, alpha = C^-1 (y - m), P = C^-1 K_xs, mu* = m* + K_sx alpha, Sigma = K_ss - K_sx P + Sigma* = L* L*'
and Obar the cotangent of out:
    Zbar = L*' Obar,  mubar = Obar 1,  Sigmabar = 1/2 V*' Q V*   (V* = L*^-1, Q = the lower triangle of Zbar Z' mirrored:
                                                                 rand_grad_ref's Cholesky pullback applied to L*)
and from Sigmabar and mubar the training side of the held-out gradient (pred_logpdf_grad_ref):
    beta = P mubar,  Kbar_sx = mubar alpha' - 2 Sigmabar P',  Cbar = P Sigmabar P' - 1/2 (beta alpha' + alpha beta')
    ybar = beta,  mbar = -beta,  mbar* = mubar,  d/d sigma_i^2 = Cbar_ii,  d/d sigma*_m^2 = Sigmabar_mm
with the kernel terms 1/2 <W, dK([x; x*])>, W = [2 Cbar, Kbar_xs; Kbar_sx, 2 Sigmabar] (rand_grad_ref.descriptor_grad)."""
import numpy as np
from scipy.linalg import cho_factor, cho_solve, solve_triangular

import composite_ref as cr
import grad_x_ref as gx
import rand_grad_ref as rg
from oracle import agp_ref as ref


def _single_layout(k, gc, D):
    """the one-factor descriptor [5] variance, [6..] Scale s | ARD v, then Linear c, in the single-kernel layout"""
    if isinstance(k, cr.Composite):
        return gc
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
    return g


def post_rand_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, Z, Obar):
    """dict: "out" (M x S), "grad" (grad_out: 5 + D for a KernelSpec, the descriptor layout for a Composite),
    "noise_diag", "mean_diag", "y" (N), "x" (N x D), "noise_s_diag", "mean_s_diag" (M), "Z" (M x S), "xs" (M x D).
    mean_s is the prior mean at Xs (a MeanSpec of the same kind as mean)."""
    X = np.asarray(X, dtype=np.float64)
    Xs = np.asarray(Xs, dtype=np.float64)
    N, D = X.shape
    M = Xs.shape[0]
    Z = np.asarray(Z, dtype=np.float64).reshape(M, -1)
    Obar = np.asarray(Obar, dtype=np.float64).reshape(M, -1)
    kc = gx.as_composite(k)
    Kxx = cr.kernelmatrix(kc, X)
    Kxs = cr.kernelmatrix(kc, X, Xs)
    Kss = cr.kernelmatrix(kc, Xs)
    cf = cho_factor(Kxx + np.diag(noise.diag(N, np.float64)), lower=True)
    alpha = cho_solve(cf, np.asarray(y, dtype=np.float64) - mean.vector(N, np.float64))
    P = cho_solve(cf, Kxs)
    mu = mean_s.vector(M, np.float64) + Kxs.T @ alpha
    Ls = np.linalg.cholesky(Kss - Kxs.T @ P + np.diag(noise_s.diag(M, np.float64)))
    out = mu[:, None] + Ls @ Z
    Zbar = Ls.T @ Obar
    Q = np.tril(Zbar @ Z.T)
    Q = Q + np.tril(Q, -1).T
    Vs = solve_triangular(Ls, np.eye(M), lower=True)
    Sbar = 0.5 * Vs.T @ Q @ Vs
    mubar = Obar.sum(axis=1)
    beta = P @ mubar
    Kbar = np.outer(mubar, alpha) - 2.0 * Sbar @ P.T
    Cbar = P @ Sbar @ P.T - 0.5 * (np.outer(beta, alpha) + np.outer(alpha, beta))
    W = np.block([[2.0 * Cbar, Kbar.T], [Kbar, 2.0 * Sbar]])
    g = _single_layout(k, rg.descriptor_grad(k, W, np.vstack([X, Xs])), D)
    g[3] = np.trace(Cbar)
    g[4] = np.sum(mubar) - np.sum(beta)
    xg = 2.0 * np.einsum("ij,ijd->id", Cbar, gx.kernel_d1(k, X, X)) + np.einsum("mi,imd->id", Kbar, gx.kernel_d1(k, X, Xs))
    xsg = 2.0 * np.einsum("ij,ijd->id", Sbar, gx.kernel_d1(k, Xs, Xs)) + np.einsum("mi,mid->md", Kbar, gx.kernel_d1(k, Xs, X))
    return {"out": out, "grad": g, "noise_diag": np.diag(Cbar).copy(), "mean_diag": -beta, "y": beta, "x": xg,
            "noise_s_diag": np.diag(Sbar).copy(), "mean_s_diag": mubar, "Z": Zbar, "xs": xsg}
