"""CPU model of the gradient of logpdf(fx, y) with respect to the input points (agp.h agp_post_logpdf_grad_x), in NumPy,
for single kernels (oracle.agp_ref.KernelSpec) and composites (tests/composite_ref.Composite).  Test infrastructure only.

    dL/dx_{i,d} = sum_j W_ij d1k(x_i, x_j)_d,   W = alpha alpha' - C^-1

d1 is the derivative in the first argument with respect to the untransformed input.  A single kernel is evaluated as a
one-factor composite; each factor forms its own transformed differences (no shared accumulators, unlike the device)."""
import numpy as np

import composite_ref as cr
from oracle import agp_ref as ref


def as_composite(k):
    """a single-kernel KernelSpec as a one-term, one-factor composite (the same kernel)"""
    if isinstance(k, cr.Composite):
        return k
    F = cr.Factor(k.family, k.transform, k.scale, k.linear_c if k.family == ref.LINEAR else 0.0,
                  None if k.ard is None else np.asarray(k.ard, dtype=np.float64))
    return cr.Composite([k.variance], [[F]])


def _t(F, D):
    if F.transform == cr.T_SCALE:
        return np.full(D, float(F.scale))
    if F.transform == cr.T_ARD:
        return np.asarray(F.ard, dtype=np.float64)
    return np.ones(D)


def factor_d1(F, XI, X):
    """d1 kappa_f(x_i, x_j) for the rows XI against all points X: (|I|, n, D); exactly 0 where x~_i == x~_j for the
    stationary factors (Matern 1/2 included: its zero subgradient)"""
    D = X.shape[1]
    t = _t(F, D)
    diff = XI[:, None, :] - X[None, :, :]
    if F.family in (cr.WHITE, cr.CONSTANT):
        return np.zeros(diff.shape)
    if F.family == cr.LINEAR:
        return np.broadcast_to((t * t) * X[None, :, :], diff.shape).copy()
    kap = cr._factor(F, XI, X, False)
    if F.family == cr.PERIODIC:
        r = np.ones(D) if F.r is None else np.asarray(F.r, dtype=np.float64)
        return kap[:, :, None] * (-np.pi * t / (2.0 * r * r)) * np.sin(np.pi * 2.0 * t * diff)
    dt = t * diff
    d2 = np.sum(dt * dt, axis=2)
    d = np.sqrt(d2)
    with np.errstate(divide="ignore", invalid="ignore"):
        if F.family == cr.SE:
            q = -np.exp(-0.5 * d2)
        elif F.family == cr.MATERN12:
            q = np.where(d > 0, -np.exp(-d) / np.where(d > 0, d, 1.0), 0.0)
        elif F.family == cr.MATERN32:
            q = -3.0 * np.exp(-np.sqrt(3.0) * d)
        elif F.family == cr.MATERN52:
            s = np.sqrt(5.0) * d
            q = -(5.0 / 3.0) * (1.0 + s) * np.exp(-s)
        else:  # RQ
            q = -kap / (1.0 + d2 / (2.0 * F.param))
    return q[:, :, None] * (t * t) * diff


def kernel_d1(k, XI, X):
    """d1 K(x_i, x_j) = sum_t v_t sum_{f in t} prod_{g != f} kappa_g d1 kappa_f: (|I|, n, D)"""
    k = as_composite(k)
    out = np.zeros((XI.shape[0], X.shape[0], X.shape[1]))
    for v, fs in zip(k.variance, k.factors):
        kaps = [cr._factor(F, XI, X, False) for F in fs]
        for j, F in enumerate(fs):
            other = np.full(kaps[0].shape, float(v))
            for i2, kp in enumerate(kaps):
                if i2 != j:
                    other = other * kp
            out += other[:, :, None] * factor_d1(F, XI, X)
    return out


def W_matrix(k, mean, noise, X, y):
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    m, C = cr.mean_and_cov_fx(k, mean, noise, X) if isinstance(k, cr.Composite) else ref.mean_and_cov_fx(k, mean, noise, X)
    U = ref.cholesky_upper(C)
    alpha = ref._U_solve(U, ref._Ut_solve(U, np.asarray(y, dtype=np.float64) - m))
    Vi = ref._Ut_solve(U, np.eye(n))
    return np.outer(alpha, alpha) - Vi.T @ Vi


def grad_x(k, mean, noise, X, y, block=128):
    """(n, D) gradient of logpdf with respect to the (untransformed) points, in fp64"""
    X = np.asarray(X, dtype=np.float64)
    W = W_matrix(k, mean, noise, X, y)
    n = X.shape[0]
    block = max(1, min(block, int(2e7 // max(1, n * X.shape[1]))))
    out = np.empty(X.shape)
    for i in range(0, n, block):
        out[i:i + block] = np.einsum("ij,ijd->id", W[i:i + block], kernel_d1(k, X[i:i + block], X))
    return out


def logpdf(k, mean, noise, X, y):
    return cr.logpdf(as_composite(k), mean, noise, np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64))
