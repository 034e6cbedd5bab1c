"""CPU model of the pullback of mean_and_var over an exact posterior, (mu*, sigma^2) of posterior(fx, y)(x*, Sigma*)
(agp.h agp_post_mean_var_grad), in NumPy fp64, for single kernels (oracle.agp_ref.KernelSpec) and composites
(tests/composite_ref.Composite).  Test infrastructure only.

With C = K_xx + Sigma_y, alpha = C^-1 (y - m), P = C^-1 K_xs, mu* = m* + K_sx alpha,
sigma^2 = diag(K_ss) - diag(K_sx P) + diag(Sigma*) and the cotangents mbar, vbar of the two outputs, the training side is
the held-out gradient's (pred_logpdf_grad_ref) at mubar = mbar and Sigmabar = diag(vbar):
    beta = P mbar,  Kbar_sx = mbar alpha' - 2 diag(vbar) P',  Cbar = P diag(vbar) P' - 1/2 (beta alpha' + alpha beta')
    ybar = beta,  mbar at x = -beta,  d/d sigma_i^2 = Cbar_ii,  d/d ConstMean c = sum mbar - sum beta
with the kernel terms 1/2 <W, dK([x; x*])>, W = [2 Cbar, Kbar_xs; Kbar_sx, 2 diag(vbar)] (rand_grad_ref.descriptor_grad),
and the test side
    xs_grad[j] = sum_n Kbar_sx[j, n] d1k(x*_j, x_n) + 2 vbar_j d1k(x*_j, x*_j),  d/d m*_j = mbar_j,  d/d sigma*_j^2 = vbar_j."""
import numpy as np
from scipy.linalg import cho_factor, cho_solve

import composite_ref as cr
import grad_x_ref as gx
import rand_grad_ref as rg
from post_rand_grad_ref import _single_layout


def post_mean_var_grad(k, mean, noise, X, y, Xs, mean_s, noise_s, mbar, vbar):
    """dict: "mean", "var" (M), "grad" (grad_out: 5 + D for a KernelSpec, the descriptor layout for a Composite) and
    "grad_abs" (the magnitudes of its kernel entries' three block terms),
    "noise_diag", "mean_diag", "y" (N), "x" (N x D), "noise_s_diag", "mean_s_diag" (M), "xs" (M x D).  mean_s is the prior
    mean at Xs (a MeanSpec of the same kind as mean)."""
    X = np.asarray(X, dtype=np.float64)
    Xs = np.asarray(Xs, dtype=np.float64)
    N, D = X.shape
    M = Xs.shape[0]
    mbar = np.asarray(mbar, dtype=np.float64).reshape(M)
    vbar = np.asarray(vbar, dtype=np.float64).reshape(M)
    kc = gx.as_composite(k)
    Kxx = cr.kernelmatrix(kc, X)
    Kxs = cr.kernelmatrix(kc, X, Xs)
    Kss = cr.kernelmatrix(kc, Xs)
    cf = cho_factor(Kxx + np.diag(noise.diag(N, np.float64)), lower=True)
    alpha = cho_solve(cf, np.asarray(y, dtype=np.float64) - mean.vector(N, np.float64))
    P = cho_solve(cf, Kxs)
    mu = mean_s.vector(M, np.float64) + Kxs.T @ alpha
    var = np.diag(Kss) - np.einsum("nj,nj->j", Kxs, P) + noise_s.diag(M, np.float64)
    beta = P @ mbar
    Kbar = np.outer(mbar, alpha) - 2.0 * vbar[:, None] * P.T
    Cbar = (P * vbar) @ P.T - 0.5 * (np.outer(beta, alpha) + np.outer(alpha, beta))
    Sbar = np.diag(vbar)
    W = np.block([[2.0 * Cbar, Kbar.T], [Kbar, 2.0 * Sbar]])
    g = _single_layout(k, rg.descriptor_grad(k, W, np.vstack([X, Xs])), D)
    g[3] = np.trace(Cbar)
    g[4] = np.sum(mbar) - np.sum(beta)
    xg = 2.0 * np.einsum("ij,ijd->id", Cbar, gx.kernel_d1(k, X, X)) + np.einsum("mi,imd->id", Kbar, gx.kernel_d1(k, X, Xs))
    d1s = gx.kernel_d1(k, Xs, Xs)
    xsg = np.einsum("mi,mid->md", Kbar, gx.kernel_d1(k, Xs, X)) + 2.0 * vbar[:, None] * d1s[np.arange(M), np.arange(M)]
    # the kernel entries' three block terms <Cbar, dK_xx>, <Kbar_sx, dK_sx>, <Sigmabar, dK_ss> in magnitude: they cancel
    # (the means barely depend on the variance), and their sum is the scale of an entry's rounding error
    g_abs = np.zeros_like(g)
    for blk in ((slice(0, N), slice(0, N)), (slice(N, None), slice(0, N)), (slice(N, None), slice(N, None))):
        Wb = np.zeros_like(W)
        Wb[blk] = W[blk]
        Wb[blk[::-1]] = W[blk[::-1]]
        g_abs += np.abs(_single_layout(k, rg.descriptor_grad(k, Wb, np.vstack([X, Xs])), D))
    return {"mean": mu, "var": var, "grad": g, "grad_abs": g_abs, "noise_diag": np.diag(Cbar).copy(), "mean_diag": -beta, "y": beta, "x": xg,
            "noise_s_diag": vbar.copy(), "mean_s_diag": mbar.copy(), "xs": xsg}
