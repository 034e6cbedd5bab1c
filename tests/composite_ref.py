"""CPU model of composite kernels (sums of product terms, agp.h agp_kernel_composite), in NumPy: the kernel matrix, its
diagonal, logpdf, the posterior and its predictions, sequential conditioning, and the logpdf gradient in the layout of
agp_post_logpdf_grad.  Test infrastructure only.

Unlike the device, which shares raw distance sums between factors, every factor here transforms the inputs itself and
forms its own distances, following the KernelFunctions definitions:
  SE / Matern    the single-kernel families (oracle.agp_ref._kappa)
  RQ             (1 + d2 / (2 alpha))^(-alpha)
  Periodic       exp(-1/2 sum_i (sinpi(x~_i - y~_i) / r_i)^2)
  White          1 if x~ == y~ else 0
  Constant       c
  Linear         x~ . y~ + c
"""
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

from oracle import agp_ref as ref

SE, MATERN12, MATERN32, MATERN52, LINEAR, RQ, PERIODIC, WHITE, CONSTANT = range(9)
T_NONE, T_SCALE, T_ARD = 0, 1, 2


@dataclass
class Factor:
    family: int
    transform: int = T_NONE
    scale: float = 1.0
    param: float = 0.0           # RQ alpha | Linear c | Constant c
    ard: Optional[np.ndarray] = None
    r: Optional[np.ndarray] = None  # Periodic, D values (None -> ones)

    def apply(self, X):
        if self.transform == T_SCALE:
            return X * X.dtype.type(self.scale)
        if self.transform == T_ARD:
            return X * np.asarray(self.ard, dtype=X.dtype)[None, :]
        return X


@dataclass
class Composite:
    variance: List[float]
    factors: List[List[Factor]]  # per term


def _sinpi(x):
    return np.sin(np.pi * x)


def _diffs(A, B):
    return A[:, None, :] - B[None, :, :]


def _factor(F: Factor, X, Z, sym):
    """(kappa_f, pieces for the gradient) for inputs X, Z (same dtype)"""
    A, B = F.apply(X), F.apply(Z)
    T = X.dtype.type
    if F.family == CONSTANT:
        return np.full((X.shape[0], Z.shape[0]), T(F.param), dtype=X.dtype)
    if F.family == LINEAR:
        return A @ B.T + T(F.param)
    if F.family == PERIODIC:
        r = np.ones(X.shape[1]) if F.r is None else np.asarray(F.r, dtype=np.float64)
        s = _sinpi(_diffs(A, B)) / r.astype(X.dtype)
        return np.exp(-T(0.5) * np.sum(s * s, axis=2))
    d2 = np.sum(_diffs(A, B) ** 2, axis=2)
    if sym:
        np.fill_diagonal(d2, 0)
    if F.family == WHITE:
        return (d2 == 0).astype(X.dtype)
    if F.family == RQ:
        a = T(F.param)
        return (T(1) + d2 / (T(2) * a)) ** (-a)
    return ref._kappa(F.family, d2)


def kernelmatrix(k: Composite, X, Z=None):
    sym = Z is None
    Z = X if Z is None else np.asarray(Z, dtype=X.dtype)
    K = np.zeros((X.shape[0], Z.shape[0]), dtype=X.dtype)
    for v, fs in zip(k.variance, k.factors):
        P = np.full(K.shape, X.dtype.type(v), dtype=X.dtype)
        for F in fs:
            P = P * _factor(F, X, Z, sym)
        K = K + P
    return K


def kernelmatrix_diag(k: Composite, X):
    return np.array([kernelmatrix(k, X[i:i + 1])[0, 0] for i in range(X.shape[0])], dtype=X.dtype)


def mean_and_cov_fx(k, mean, noise, X):
    n = X.shape[0]
    C = kernelmatrix(k, X)
    C[np.diag_indices(n)] += noise.diag(n, X.dtype)
    return mean.vector(n, X.dtype), C


def logpdf(k, mean, noise, X, Y):
    dtype = X.dtype
    Y = np.asarray(Y, dtype=dtype)
    m, C = mean_and_cov_fx(k, mean, noise, X)
    U = ref.cholesky_upper(C)
    n = X.shape[0]
    sq = ref.tr_Xt_invA_X(U, Y - m) if Y.ndim == 1 else ref.diag_Xt_invA_X(U, Y - m[:, None])
    return -((n * dtype.type(ref.LOG2PI) + dtype.type(ref.logdet_chol(U))) + sq) / dtype.type(2)


def posterior(k, mean, noise, X, y):
    m, C = mean_and_cov_fx(k, mean, noise, X)
    U = ref.cholesky_upper(C)
    delta = np.asarray(y, dtype=X.dtype) - m
    alpha = ref._U_solve(U, ref._Ut_solve(U, delta))
    return dict(alpha=alpha, U=U, x=X, delta=delta, k=k, mean=mean)


def post_mean_and_var(post, Xs, noise_s=None):
    k, X = post["k"], post["x"]
    Xs = np.asarray(Xs, dtype=X.dtype)
    Kxs = kernelmatrix(k, X, Xs)
    m = post["mean"].vector(Xs.shape[0], X.dtype) + Kxs.T @ post["alpha"]
    v = kernelmatrix_diag(k, Xs) - ref.diag_Xt_invA_X(post["U"], Kxs)
    if noise_s is not None:
        v = v + noise_s.diag(Xs.shape[0], X.dtype)
    return m, v


def post_mean_and_cov(post, Xs):
    k, X = post["k"], post["x"]
    Xs = np.asarray(Xs, dtype=X.dtype)
    Kxs = kernelmatrix(k, X, Xs)
    m = post["mean"].vector(Xs.shape[0], X.dtype) + Kxs.T @ post["alpha"]
    return m, kernelmatrix(k, Xs) - ref.Xt_invA_X(post["U"], Kxs)


def post_logpdf(post, Xs, noise_s, Y):
    dtype = post["x"].dtype
    m, C = post_mean_and_cov(post, Xs)
    n = C.shape[0]
    C[np.diag_indices(n)] += noise_s.diag(n, dtype)
    U = ref.cholesky_upper(C)
    Y = np.asarray(Y, dtype=dtype)
    sq = ref.tr_Xt_invA_X(U, Y - m) if Y.ndim == 1 else ref.diag_Xt_invA_X(U, Y - m[:, None])
    return -((n * dtype.type(ref.LOG2PI) + dtype.type(ref.logdet_chol(U))) + sq) / dtype.type(2)


def post_rand_from_Z(post, Xs, noise_s, Z):
    m, C = post_mean_and_cov(post, Xs)
    n = C.shape[0]
    C[np.diag_indices(n)] += noise_s.diag(n, post["x"].dtype)
    U = ref.cholesky_upper(C)
    return m[:, None] + U.T @ np.asarray(Z, dtype=post["x"].dtype)


def posterior_sequential(post, noise2, X2, y2):
    k, X1 = post["k"], post["x"]
    X2 = np.asarray(X2, dtype=X1.dtype)
    d2 = np.asarray(y2, dtype=X1.dtype) - post["mean"].vector(X2.shape[0], X1.dtype)
    C22 = kernelmatrix(k, X2)
    C22[np.diag_indices(X2.shape[0])] += noise2.diag(X2.shape[0], X1.dtype)
    U = ref.update_chol(post["U"], kernelmatrix(k, X1, X2), C22)
    delta = np.concatenate([post["delta"], d2])
    alpha = ref._U_solve(U, ref._Ut_solve(U, delta))
    return dict(alpha=alpha, U=U, x=np.concatenate([X1, X2], 0), delta=delta, k=k, mean=post["mean"])


# ---- gradient ------------------------------------------------------------------------------------------------------
def grad_len(k: Composite, D):
    n = 5
    for fs in k.factors:
        n += 1
        for F in fs:
            n += 1 if F.transform == T_SCALE else (D if F.transform == T_ARD else 0)
            n += 1 if F.family in (RQ, LINEAR, CONSTANT) else 0
            n += D if F.family == PERIODIC else 0
    return n


def _factor_derivs(F: Factor, X):
    """[(kind, dK_f/dtheta)] in the ABI order of the factor's slots: Scale s or ARD v_d, then param, then r_d"""
    D = X.shape[1]
    A = F.apply(X)
    kap = _factor(F, X, X, True)
    out = []
    diff = _diffs(X, X)  # untransformed
    w = np.full(D, F.scale) if F.transform != T_ARD else np.asarray(F.ard, dtype=np.float64)
    if F.transform == T_NONE:
        w = np.ones(D)
    if F.family == PERIODIC:
        r = np.ones(D) if F.r is None else np.asarray(F.r, dtype=np.float64)
        arg = w[None, None, :] * diff
        sn, cs = _sinpi(arg), np.cos(np.pi * arg)
        dw = -kap[:, :, None] * np.pi * diff * sn * cs / r ** 2     # d kappa / d w_d
        if F.transform == T_SCALE:
            out.append(dw.sum(axis=2))
        elif F.transform == T_ARD:
            out += [dw[:, :, d] for d in range(D)]
        out += [kap * sn[:, :, d] ** 2 / r[d] ** 3 for d in range(D)]
        return out
    if F.family in (CONSTANT, WHITE):
        if F.transform == T_SCALE:
            out.append(np.zeros_like(kap))
        elif F.transform == T_ARD:
            out += [np.zeros_like(kap)] * D
        if F.family == CONSTANT:
            out.append(np.ones_like(kap))
        return out
    if F.family == LINEAR:
        G = X @ X.T
        if F.transform == T_SCALE:
            out.append(2.0 * F.scale * G)
        elif F.transform == T_ARD:
            out += [2.0 * w[d] * np.outer(X[:, d], X[:, d]) for d in range(D)]
        out.append(np.ones_like(kap))
        return out
    d2 = np.sum(_diffs(A, A) ** 2, axis=2)
    np.fill_diagonal(d2, 0)
    if F.family == RQ:
        u = d2 / (2.0 * F.param)
        q = -kap / (1.0 + u)                                         # 2 d kappa / d d2
    else:
        with np.errstate(divide="ignore", invalid="ignore"):
            q = np.where(d2 > 0, ref._dkappa_r(F.family, d2) / d2, 0.0)
    if F.transform == T_SCALE:
        out.append(q * F.scale * np.sum(diff ** 2, axis=2))
    elif F.transform == T_ARD:
        out += [q * w[d] * diff[:, :, d] ** 2 for d in range(D)]
    if F.family == RQ:
        out.append(kap * (u / (1.0 + u) - np.log1p(u)))
    return out


def logpdf_grad(k: Composite, mean, noise, X, y):
    """(descriptor gradient in the agp_post_logpdf_grad layout, noise gradient: scalar or per point)"""
    X = np.asarray(X, dtype=np.float64)
    n, D = X.shape
    m, C = mean_and_cov_fx(k, mean, noise, X)
    U = ref.cholesky_upper(C)
    alpha = ref._U_solve(U, ref._Ut_solve(U, np.asarray(y, dtype=np.float64) - m))
    Vi = ref._Ut_solve(U, np.eye(n))
    W = np.outer(alpha, alpha) - Vi.T @ Vi
    g = np.zeros(grad_len(k, D))
    g[3] = 0.5 * np.trace(W)
    g[4] = np.sum(alpha)
    pos = 5
    for v, fs in zip(k.variance, k.factors):
        kaps = [_factor(F, X, X, True) for F in fs]
        g[pos] = 0.5 * np.sum(W * np.prod(kaps, axis=0))
        pos += 1
        for j, F in enumerate(fs):
            other = v * np.prod([kaps[i] for i in range(len(fs)) if i != j], axis=0) if len(fs) > 1 else v
            for dK in _factor_derivs(F, X):
                g[pos] = 0.5 * np.sum(W * other * dK)
                pos += 1
    assert pos == len(g)
    return g, (0.5 * np.trace(W) if noise.kind == 0 else 0.5 * np.diag(W).copy())


def from_struct(ks, D, dt):
    """Composite from a ctypes agp_kernel with family AGP_COMPOSITE (the descriptor a caller passes the library)"""
    import ctypes as C

    def arr(p):
        if not p:
            return None
        ct = C.c_double if np.dtype(dt) == np.float64 else C.c_float
        return np.array(np.ctypeslib.as_array((ct * D).from_address(p)), dtype=np.float64)
    c = ks.composite.contents
    variance, factors, f = [], [], 0
    for t in range(c.nterms):
        variance.append(c.variance[t])
        fs = []
        for _ in range(c.nfactors[t]):
            fa = c.factors[f]
            fs.append(Factor(fa.family, fa.transform, fa.scale, fa.param, arr(fa.ard), arr(fa.r)))
            f += 1
        factors.append(fs)
    return Composite(variance, factors)
