"""CPU model of the pullback of rand(fx, S) (agp.h agp_rand_grad), in NumPy fp64, for single kernels
(oracle.agp_ref.KernelSpec) and composites (tests/composite_ref.Composite).  Test infrastructure only.

With out = m + L Z, C = K + Sigma_y = L L' and Obar the cotangent of out:
    Zbar = L' Obar,  mbar = Obar 1,  W = 2 Cbar = V' Q V  (V = L^-1, Q = the lower triangle of Zbar Z' mirrored)
and from W the reductions of the logpdf gradient: d/d theta = 1/2 sum W o dK/dtheta, d/d sigma^2 = 1/2 tr W (per point
1/2 W_ii), dx_i = sum_j W_ij d1k(x_i, x_j)."""
import numpy as np

import composite_ref as cr
import grad_x_ref as gx
from oracle import agp_ref as ref


def W_matrix(k, mean, noise, X, Z, Obar):
    """(W = 2 Cbar, Zbar, mbar) in fp64; Z and Obar are N x S"""
    X = np.asarray(X, dtype=np.float64)
    kc = gx.as_composite(k)
    m, C = cr.mean_and_cov_fx(kc, mean, noise, X)
    U = ref.cholesky_upper(C)  # L = U'
    Z = np.asarray(Z, dtype=np.float64).reshape(X.shape[0], -1)
    Obar = np.asarray(Obar, dtype=np.float64).reshape(X.shape[0], -1)
    Zbar = U @ Obar
    P = Zbar @ Z.T
    Q = np.tril(P) + np.tril(P, -1).T
    V = ref._Ut_solve(U, np.eye(X.shape[0]))
    return V.T @ Q @ V, Zbar, Obar.sum(axis=1)


def descriptor_grad(k, W, X):
    """1/2 sum_ij W_ij dK_ij/dtheta in the agp_post_logpdf_grad layout of the composite form of k ([3], [4] left 0)"""
    X = np.asarray(X, dtype=np.float64)
    kc = gx.as_composite(k)
    g = np.zeros(cr.grad_len(kc, X.shape[1]))
    pos = 5
    for v, fs in zip(kc.variance, kc.factors):
        kaps = [cr._factor(F, X, X, True) for F in fs]
        g[pos] = 0.5 * np.sum(W * np.prod(kaps, axis=0))
        pos += 1
        for j, F in enumerate(fs):
            other = v * np.prod([kaps[i] for i in range(len(fs)) if i != j], axis=0) if len(fs) > 1 else v
            for dK in cr._factor_derivs(F, X):
                g[pos] = 0.5 * np.sum(W * other * dK)
                pos += 1
    assert pos == len(g)
    return g


def rand_grad(k, mean, noise, X, Z, Obar):
    """dict: "grad" (agp_rand_grad's grad_out: 5 + D for a KernelSpec, the descriptor layout for a Composite),
    "noise_diag", "mean_diag", "x" (N x D), "Z" (N x S)"""
    X = np.asarray(X, dtype=np.float64)
    n, D = X.shape
    W, Zbar, mbar = W_matrix(k, mean, noise, X, Z, Obar)
    gc = descriptor_grad(k, W, X)
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
    g[3] = 0.5 * np.trace(W)
    g[4] = np.sum(mbar)
    xg = np.empty(X.shape)
    block = max(1, min(128, int(2e7 // max(1, n * D))))
    for i in range(0, n, block):
        xg[i:i + block] = np.einsum("ij,ijd->id", W[i:i + block], gx.kernel_d1(k, X[i:i + block], X))
    return {"grad": g, "noise_diag": 0.5 * np.diag(W).copy(), "mean_diag": mbar, "x": xg, "Z": Zbar}


def rand(k, mean, noise, X, Z):
    """out = m + C.U' Z in fp64 (oracle.agp_ref.rand_from_Z for composites too)"""
    X = np.asarray(X, dtype=np.float64)
    m, C = cr.mean_and_cov_fx(gx.as_composite(k), mean, noise, X)
    U = ref.cholesky_upper(C)
    return m[:, None] + U.T @ np.asarray(Z, dtype=np.float64).reshape(X.shape[0], -1)
