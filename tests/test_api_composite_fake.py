"""The host mirror's composite kernels (abstractgps.jl_b200/api.py: KernelSum / KernelProduct, flattening into the
agp_kernel_composite descriptor, kernel_params and the chain rule of logpdf_grad) driven on the CPU through a stand-in
library that reads the descriptor with the composite model (tests/composite_ref.py)."""
import ctypes as C

import numpy as np
import pytest

import composite_ref as cr
import fake_libagp
from oracle import agp_ref as ref


class CompositeFakeLib(fake_libagp.FakeLib):
    """FakeLib that answers AGP_COMPOSITE kernels with the composite model"""

    def _kernel(self, ks, D, dt):
        s = fake_libagp._struct(ks)
        if s.family == 9:
            return cr.from_struct(s, D, dt)
        return super()._kernel(ks, D, dt)

    def agp_gram(self, h, code, ks, layout, X, n, D, Z, m, ns, K_out):
        dt = self._dt(code)
        k = self._kernel(ks, D, dt)
        if not isinstance(k, cr.Composite):
            return super().agp_gram(h, code, ks, layout, X, n, D, Z, m, ns, K_out)
        Xa = self._points(layout, X, n, D, dt)
        if fake_libagp._addr(Z) is None:
            K = cr.kernelmatrix(k, Xa)
            if fake_libagp._struct(ns) is not None:
                K[np.diag_indices(n)] += self._noise(ns, n, dt).diag(n, dt)
            fake_libagp._arr(K_out, (n, n), dt, "F")[...] = K
        else:
            fake_libagp._arr(K_out, (n, m), dt, "F")[...] = cr.kernelmatrix(k, Xa, self._points(layout, Z, m, D, dt))
        return 0

    def agp_fit(self, h, code, ks, ms, ns, layout, X, n, D, Y, S, lp_out, alpha_out, post_out):
        dt = self._dt(code)
        k = self._kernel(ks, D, dt)
        if not isinstance(k, cr.Composite):
            return super().agp_fit(h, code, ks, ms, ns, layout, X, n, D, Y, S, lp_out, alpha_out, post_out)
        mean, noise = self._mean(ms, n, dt), self._noise(ns, n, dt)
        Xa = self._points(layout, X, n, D, dt)
        Ya = np.array(fake_libagp._arr(Y, (n, S), dt, "F"))
        fake_libagp._arr(lp_out, (S,), dt)[...] = cr.logpdf(k, mean, noise, Xa, Ya)
        post = cr.posterior(k, mean, noise, Xa, Ya[:, 0])
        if fake_libagp._addr(alpha_out) is not None:
            fake_libagp._arr(alpha_out, (n,), dt)[...] = post["alpha"]
        if post_out is not None:
            post["noise"] = noise
            post_out._obj.value = self._new(self.posts, post)
        return 0

    def agp_post_grad_len(self, p):
        post = self.posts[self._h(p)]
        return cr.grad_len(post["k"], post["x"].shape[1])

    def agp_post_logpdf_grad(self, p, grad_out, noise_diag_out):
        post = self.posts[self._h(p)]
        X = post["x"].astype(np.float64)
        y = post["delta"] + post["mean"].vector(X.shape[0], np.float64)
        g, gn = cr.logpdf_grad(post["k"], post["mean"], ref.NoiseSpec(1, v=post["noise"].diag(X.shape[0], np.float64)), X, y)
        np.ctypeslib.as_array(grad_out, shape=(len(g),))[:] = g
        if fake_libagp._addr(noise_diag_out) is not None:
            fake_libagp._arr(noise_diag_out, (X.shape[0],), post["x"].dtype)[...] = gn
        return 0


@pytest.fixture
def fake(ag, monkeypatch):
    eng = ag.api.Engine.__new__(ag.api.Engine)
    eng.L, eng.h, eng.device = CompositeFakeLib(), C.c_void_p(1), 0
    monkeypatch.setattr(ag.api, "_engine", eng)
    return eng


def tree_K(ag, k, X, Z=None):
    """the kernel tree evaluated node by node (no flattening): sums add, products multiply, scalings scale, a node's
    transform is applied to its inputs before its children see them"""
    sym = Z is None
    Z = X if Z is None else Z
    t = k.transform
    if t is not None:
        w = t.s if isinstance(t, ag.ScaleTransform) else t.v[None, :]
        X, Z = X * w, Z * w
    if isinstance(k, ag.KernelSum):
        K = sum(tree_K(ag, ch, X, None if sym else Z) for ch in k.kernels)
    elif isinstance(k, ag.KernelProduct):
        K = np.prod([tree_K(ag, ch, X, None if sym else Z) for ch in k.kernels], axis=0)
    else:
        param = k.alpha if k.family == ag.api.RQ else k.c
        K = cr._factor(cr.Factor(k.family, param=param, r=None if k.r is None else np.broadcast_to(k.r, (X.shape[1],))),
                       X, Z, sym)
    return k.variance * K


def kernels(ag):
    SE, Per = ag.SqExponentialKernel, ag.PeriodicKernel
    s = 0.7 * ag.with_lengthscale(SE() + 2.0 * ag.Matern32Kernel(), 1.5)          # scaled, transformed sum
    return {
        "nested": (SE() + (ag.Matern12Kernel() + 0.5 * ag.RationalQuadraticKernel(1.2))) * Per(r=[0.8]),
        "scaled_transformed_sum": s + ag.WhiteKernel(),
        "product_over_sum": ag.with_lengthscale(Per(r=[1.1, 0.6]), [1.3, 0.7]) * s + ag.LinearKernel(c=0.2) * s,
        "ard_chain": ag.SqExponentialKernel().compose(ag.ARDTransform([0.5, 2.0])).compose(ag.ScaleTransform(0.8))
        + ag.RationalQuadraticKernel(0.7) * ag.LinearKernel(0.4).compose(ag.ARDTransform([1.0, 0.3])),
        # a leaf built with a variance (not through sigma^2 * k) keeps it inside a sum / product
        "unscaled_variance": ag.api.Kernel(ag.api.SE, variance=2.0) * ag.PeriodicKernel(r=[0.9])
        + ag.api.Kernel(ag.api.MATERN52, variance=0.5, transform=ag.ScaleTransform(0.7)),
    }


@pytest.mark.parametrize("name", ["nested", "scaled_transformed_sum", "product_over_sum", "ard_chain", "unscaled_variance"])
def test_flattening_matches_tree(ag, fake, name):
    k = kernels(ag)[name]
    rng = np.random.default_rng(0)
    X, Z = rng.normal(size=(15, 2)), rng.normal(size=(9, 2))
    X[7] = X[3]  # a duplicate for White
    np.testing.assert_allclose(ag.kernelmatrix(k, ag.RowVecs(X)), tree_K(ag, k, X), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(ag.kernelmatrix(k, ag.RowVecs(X), ag.RowVecs(Z)), tree_K(ag, k, X, Z), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(ag.var(ag.GP(k), ag.RowVecs(Z)), np.diag(tree_K(ag, k, Z)), rtol=1e-13, atol=1e-13)


def test_limits_raise(ag, fake):
    three = ag.SqExponentialKernel() + ag.Matern12Kernel() + ag.Matern32Kernel()
    with pytest.raises(ag.AGPError) as e:
        ag.kernelmatrix(three * three, np.linspace(0, 1, 4))  # 9 terms
    assert e.value.code == ag._cabi.AGP_ERR_UNSUPPORTED
    many = ag.SqExponentialKernel()
    for _ in range(8):
        many = many * ag.Matern52Kernel()  # 9 factors
    with pytest.raises(ag.AGPError):
        ag.kernelmatrix(many, np.linspace(0, 1, 4))


@pytest.mark.parametrize("name", ["nested", "scaled_transformed_sum", "product_over_sum", "ard_chain", "unscaled_variance"])
def test_logpdf_grad_in_kernel_params_order(ag, fake, name):
    """out["kernel"] equals central differences of logpdf in kernel_params(k) order, shared parameters included"""
    k = kernels(ag)[name]
    rng = np.random.default_rng(1)
    X = rng.normal(size=(20, 2))
    y = rng.normal(size=20)
    s2 = 0.3
    lp, g = ag.logpdf_grad(ag.GP(0.2, k)(ag.RowVecs(X), s2), y)
    vals = ag.kernel_params(k)
    assert len(g["kernel"]) == len(vals)
    h = 1e-6

    def L(v):
        return ag.logpdf(ag.GP(0.2, ag.with_kernel_params(k, v))(ag.RowVecs(X), s2), y)
    for i, v in enumerate(vals):
        for j in range(np.size(v)):
            vp = [np.array(x, dtype=float) if np.ndim(x) else x for x in vals]
            vm = [np.array(x, dtype=float) if np.ndim(x) else x for x in vals]
            if np.ndim(v):
                vp[i][j] += h
                vm[i][j] -= h
            else:
                vp[i] += h
                vm[i] -= h
            fd = (L(vp) - L(vm)) / (2 * h)
            gi = g["kernel"][i][j] if np.ndim(v) else g["kernel"][i]
            assert abs(gi - fd) <= 1e-6 * max(1.0, abs(fd)), (name, i, j, gi, fd)
    fdn = (ag.logpdf(ag.GP(0.2, k)(ag.RowVecs(X), s2 + h), y) - ag.logpdf(ag.GP(0.2, k)(ag.RowVecs(X), s2 - h), y)) / (2 * h)
    assert abs(g["noise"] - fdn) <= 1e-6 * max(1.0, abs(fdn))
