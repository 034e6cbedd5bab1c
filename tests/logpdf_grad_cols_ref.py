"""CPU model of the gradient of sum_s w_s logpdf(fx, Y[:, s]) for a matrix Y (agp.h agp_post_logpdf_grad_cols), in NumPy
fp64, for single kernels (oracle.agp_ref.KernelSpec) and composites (tests/composite_ref.Composite).  Test infrastructure
only.

With delta_s = Y[:, s] - m, A = C^-1 [delta_1 .. delta_S] (by cho_solve) and w the cotangent of the S logpdfs:
    W = A diag(w) A' - (sum_s w_s) C^-1
and from W the reductions of the logpdf gradient: d/d theta = 1/2 sum W o dK/dtheta (rand_grad_ref.descriptor_grad),
d/d sigma^2 = 1/2 tr W (per point 1/2 W_ii), dx_i = sum_j W_ij d1k(x_i, x_j) (grad_x_ref), mbar = A w, Ybar = -A diag(w)."""
import numpy as np
from scipy.linalg import cho_factor, cho_solve

import composite_ref as cr
import grad_x_ref as gx
import rand_grad_ref as rg
from oracle import agp_ref as ref


def W_matrix(k, mean, noise, X, Y, w):
    """(W, A) in fp64; Y is N x S, w has S entries"""
    X = np.asarray(X, dtype=np.float64)
    m, C = cr.mean_and_cov_fx(gx.as_composite(k), mean, noise, X)
    Y = np.asarray(Y, dtype=np.float64).reshape(X.shape[0], -1)
    cf = cho_factor(C, lower=True)
    A = cho_solve(cf, Y - m[:, None])
    Cinv = cho_solve(cf, np.eye(X.shape[0]))
    w = np.asarray(w, dtype=np.float64)
    return (A * w) @ A.T - np.sum(w) * Cinv, A


def logpdf_grad_cols(k, mean, noise, X, Y, w=None):
    """dict: "grad" (grad_out: 5 + D for a KernelSpec, the descriptor layout for a Composite), "noise_diag",
    "mean_diag", "x" (N x D), "Y" (N x S)"""
    X = np.asarray(X, dtype=np.float64)
    n, D = X.shape
    Y = np.asarray(Y, dtype=np.float64).reshape(n, -1)
    w = np.ones(Y.shape[1]) if w is None else np.asarray(w, dtype=np.float64)
    W, A = W_matrix(k, mean, noise, X, Y, w)
    gc = rg.descriptor_grad(k, W, X)
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
    mbar = A @ w
    g[3] = 0.5 * np.trace(W)
    g[4] = np.sum(mbar)
    xg = np.empty(X.shape)
    block = max(1, min(128, int(2e7 // max(1, n * D))))
    for i in range(0, n, block):
        xg[i:i + block] = np.einsum("ij,ijd->id", W[i:i + block], gx.kernel_d1(k, X[i:i + block], X))
    return {"grad": g, "noise_diag": 0.5 * np.diag(W).copy(), "mean_diag": mbar, "x": xg, "Y": -A * w}
