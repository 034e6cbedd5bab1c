"""Host-side mirror of the AbstractGPs.jl public surface for the dense hot path.

Julia is not available in this image, so the reference-facing host code is written in Python with
the reference's names and argument meaning (GP, f(x, s2)::FiniteGP, logpdf, posterior,
mean_and_var, rand, VFE/elbo ...).  Every method below forwards to ONE C-ABI entry point of
libagp.so (include/agp.h); no arithmetic on N-sized data happens on the host, and nothing falls back
to a CPU implementation.  Reference citations are relative to /root/reference.
"""
from __future__ import annotations

import ctypes as C
import os
from collections import namedtuple
from typing import Optional

import numpy as np

from . import _cabi as cabi
from ._cabi import AGPError, DimensionMismatch, PosDefException  # noqa: F401

# ---------------------------------------------------------------------------------------------
# KernelFunctions.jl surface that AbstractGPs re-exports (src/AbstractGPs.jl:8)
# ---------------------------------------------------------------------------------------------
SE, MATERN12, MATERN32, MATERN52, LINEAR = range(5)
RQ, PERIODIC, WHITE, CONSTANT = cabi.AGP_RQ, cabi.AGP_PERIODIC, cabi.AGP_WHITE, cabi.AGP_CONSTANT


class Transform:
    pass


class ScaleTransform(Transform):
    def __init__(self, s: float):
        self.s = float(s)


class ARDTransform(Transform):
    def __init__(self, v):
        self.v = np.ascontiguousarray(v, dtype=np.float64).ravel()


class Kernel:
    """sigma_f^2 * (kappa o transform) -- the kernel set the engine implements on device.  RationalQuadratic (alpha),
    Periodic (r), White and Constant (c) are valid only inside a sum or product (KernelSum / KernelProduct)."""

    def __init__(self, family, variance=1.0, transform: Optional[Transform] = None, c=0.0, alpha=2.0, r=None,
                 scaled=False):
        self.family, self.variance, self.transform, self.c = family, float(variance), transform, float(c)
        self.alpha = float(alpha)
        self.r = None if r is None else np.ascontiguousarray(r, dtype=np.float64).ravel()
        self.scaled = scaled  # built as sigma^2 * k: sigma^2 is a parameter of the tree (kernel_params)

    def _copy(self, variance=None, transform=None, scaled=None):
        return Kernel(self.family, self.variance if variance is None else variance,
                      self.transform if transform is None else transform, self.c, self.alpha, self.r,
                      self.scaled if scaled is None else scaled)

    def __rmul__(self, s):  # sigma^2 * k  (ScaledKernel)
        return self._copy(variance=self.variance * float(s), scaled=True)

    def __mul__(self, o):  # k1 * k2 (KernelProduct); k * sigma^2 (ScaledKernel)
        if isinstance(o, Kernel):
            return KernelProduct(self, o)
        return self.__rmul__(o)

    def __add__(self, o):  # k1 + k2 (KernelSum)
        if not isinstance(o, Kernel):
            return NotImplemented
        return KernelSum(self, o)

    def compose(self, t: Transform):  # k o t  (TransformedKernel)
        if self.transform is not None:
            t = _chain(self.transform, t)
        return self._copy(transform=t)

    __matmul__ = compose

    def __eq__(self, o):
        return isinstance(o, Kernel) and self._key() == o._key()

    def _key(self):
        t = self.transform
        tk = None if t is None else (("s", t.s) if isinstance(t, ScaleTransform) else ("a", tuple(t.v)))
        return (self.family, self.variance, tk, self.c, self.alpha, None if self.r is None else tuple(self.r))

    __hash__ = None


def _chain(outer: Transform, inner: Transform) -> Transform:
    """(k o outer) o inner applies inner first: x -> outer(inner(x)); both are diagonal scalings."""
    if isinstance(outer, ScaleTransform) and isinstance(inner, ScaleTransform):
        return ScaleTransform(outer.s * inner.s)
    ov = outer.v if isinstance(outer, ARDTransform) else outer.s
    iv = inner.v if isinstance(inner, ARDTransform) else inner.s
    return ARDTransform(np.asarray(ov) * np.asarray(iv))


def SqExponentialKernel():
    return Kernel(SE)


SEKernel = RBFKernel = GaussianKernel = SqExponentialKernel


def Matern12Kernel():
    return Kernel(MATERN12)


ExponentialKernel = Matern12Kernel


def Matern32Kernel():
    return Kernel(MATERN32)


def Matern52Kernel():
    return Kernel(MATERN52)


def LinearKernel(c: float = 0.0):
    return Kernel(LINEAR, c=c)


def TransformedKernel(k: Kernel, t: Transform):
    return k.compose(t)


def ScaledKernel(k: Kernel, s2: float):
    return s2 * k


def with_lengthscale(k: Kernel, ell):
    """with_lengthscale(k, l) = k o ScaleTransform(1/l); vector l -> ARDTransform(1 ./ l)."""
    if np.ndim(ell) == 0:
        return k.compose(ScaleTransform(1.0 / float(ell)))
    return k.compose(ARDTransform(1.0 / np.asarray(ell, dtype=np.float64)))


def RationalQuadraticKernel(alpha: float = 2.0):
    """(1 + d^2 / (2 alpha))^(-alpha); a factor of a composite kernel."""
    return Kernel(RQ, alpha=alpha)


def PeriodicKernel(r=(1.0,)):
    """exp(-1/2 sum_i (sinpi(x_i - y_i) / r_i)^2); a factor of a composite kernel.  A length-1 r applies to every
    dimension."""
    return Kernel(PERIODIC, r=r)


def WhiteKernel():
    """1 if the (transformed) inputs are equal, else 0; a factor of a composite kernel."""
    return Kernel(WHITE)


def ConstantKernel(c: float = 1.0):
    """c; a factor of a composite kernel."""
    return Kernel(CONSTANT, c=c)


class _CompositeKernel(Kernel):
    """A sum or product of kernels, itself optionally scaled (sigma^2 * k) and transformed (k o t).  Scaling or
    transforming it applies to every leaf, as in KernelFunctions; flattening (_Flat) carries that out."""

    def __init__(self, *kernels, variance=1.0, transform=None, scaled=False):
        self.kernels = []
        for k in kernels:  # (k1 + k2) + k3 is one sum of three, like KernelFunctions' KernelSum
            if type(k) is type(self) and not k.scaled and k.transform is None:
                self.kernels.extend(k.kernels)
            else:
                self.kernels.append(k)
        self.family, self.variance, self.transform, self.scaled = cabi.AGP_COMPOSITE, float(variance), transform, scaled
        self.c, self.alpha, self.r = 0.0, 2.0, None

    def _copy(self, variance=None, transform=None, scaled=None):
        out = type(self).__new__(type(self))
        out.__dict__.update(self.__dict__)
        out.kernels = list(self.kernels)
        if variance is not None:
            out.variance = variance
        if transform is not None:
            out.transform = transform
        if scaled is not None:
            out.scaled = scaled
        return out

    def _key(self):
        t = self.transform
        tk = None if t is None else (("s", t.s) if isinstance(t, ScaleTransform) else ("a", tuple(t.v)))
        return (type(self).__name__, self.variance, tk, tuple(k._key() for k in self.kernels))


class KernelSum(_CompositeKernel):
    """k1 + k2 + ..."""


class KernelProduct(_CompositeKernel):
    """k1 * k2 * ..."""


def _walk(k: Kernel, vals: list):
    """Depth-first: register k's parameters in `vals` (scaling, transform, then the family's own) and return its terms:
    [(scaling parameter indices, [factor, ...])], a factor being a dict with its family and the indices of its
    transforms (innermost first), parameter and r."""
    sc = []
    if k.scaled or k.variance != 1.0:  # Kernel(family, variance=v) carries its variance like a ScaledKernel
        vals.append(k.variance)
        sc = [len(vals) - 1]
    tr = []
    if k.transform is not None:
        t = k.transform
        vals.append(t.s if isinstance(t, ScaleTransform) else np.array(t.v, dtype=np.float64))
        tr = [len(vals) - 1]
    if isinstance(k, KernelSum):
        terms = [tm for ch in k.kernels for tm in _walk(ch, vals)]
    elif isinstance(k, KernelProduct):
        terms = [([], [])]
        for ch in k.kernels:  # a product over a sum is distributed
            ct = _walk(ch, vals)
            terms = [(a[0] + b[0], a[1] + b[1]) for a in terms for b in ct]
    else:
        f = dict(family=k.family, tr=[], p=None, r=None)
        if k.family == RQ:
            vals.append(k.alpha)
            f["p"] = len(vals) - 1
        elif k.family in (LINEAR, CONSTANT):
            vals.append(k.c)
            f["p"] = len(vals) - 1
        if k.family == PERIODIC:
            vals.append(np.array(k.r if k.r is not None else [1.0], dtype=np.float64))
            f["r"] = len(vals) - 1
        terms = [([], [f])]
    return [(sc + s_, [dict(f, tr=f["tr"] + tr) for f in fs]) for s_, fs in terms]


def _prod_except(vals, idx, skip, D=None):
    """prod of vals[i] for i in idx except position `skip` (no division by a parameter); vectors broadcast to D"""
    out = 1.0 if D is None else np.ones(D)
    for j, i in enumerate(idx):
        if j != skip:
            out = out * (vals[i] if D is None or np.ndim(vals[i]) == 0 else np.broadcast_to(vals[i], (D,)))
    return out


class _Flat:
    """A kernel tree flattened into the engine's sum of product terms, with what the chain rule needs to map the
    descriptor's gradient back onto kernel_params(k)."""

    def __init__(self, k: Kernel, D: int):
        self.vals = []
        self.terms = _walk(k, self.vals)
        self.D = D
        nf = sum(len(fs) for _, fs in self.terms)
        if len(self.terms) > cabi.AGP_COMPOSITE_MAX or nf > cabi.AGP_COMPOSITE_MAX:
            raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "composite kernel flattens to %d terms and %d factors; the device "
                           "takes at most %d of each" % (len(self.terms), nf, cabi.AGP_COMPOSITE_MAX))
        for _, fs in self.terms:
            for f in fs:
                for i in f["tr"] + ([f["r"]] if f["r"] is not None else []):
                    if np.ndim(self.vals[i]) and self.vals[i].shape[0] not in (1, D):
                        raise DimensionMismatch("a per-dimension kernel parameter has length %d, inputs have D=%d"
                                                % (self.vals[i].shape[0], D))

    def transform_of(self, f):
        """(AGP_T_*, s, v) of factor f: its transform chain multiplied out"""
        if not f["tr"]:
            return 0, 1.0, None
        if all(np.ndim(self.vals[i]) == 0 for i in f["tr"]):
            return 1, float(np.prod([self.vals[i] for i in f["tr"]])), None
        return 2, 1.0, _prod_except(self.vals, f["tr"], -1, self.D)

    def struct(self, dt, keep):
        nt = len(self.terms)
        facs = [f for _, fs in self.terms for f in fs]
        nfa = (C.c_int32 * nt)(*[len(fs) for _, fs in self.terms])
        var = (C.c_double * nt)(*[float(_prod_except(self.vals, s_, -1)) for s_, _ in self.terms])
        fa = (cabi.agp_kernel_factor * len(facs))()
        for j, f in enumerate(facs):
            kind, s, v = self.transform_of(f)
            fa[j].family, fa[j].transform, fa[j].scale = f["family"], kind, s
            fa[j].param = float(self.vals[f["p"]]) if f["p"] is not None else 0.0
            if v is not None:
                a = np.ascontiguousarray(v, dtype=dt)
                keep.append(a)
                fa[j].ard = a.ctypes.data
            if f["r"] is not None:
                a = np.ascontiguousarray(np.broadcast_to(self.vals[f["r"]], (self.D,)), dtype=dt)
                keep.append(a)
                fa[j].r = a.ctypes.data
        comp = cabi.agp_kernel_composite()
        comp.nterms, comp.nfactors, comp.variance = nt, nfa, var
        comp.factors = C.cast(fa, C.POINTER(cabi.agp_kernel_factor))
        keep.extend([nfa, var, fa, comp])
        ks = cabi.agp_kernel()
        ks.family, ks.transform, ks.variance, ks.scale = cabi.AGP_COMPOSITE, 0, 1.0, 1.0
        ks.composite = C.pointer(comp)
        return ks

    def grad_len(self):
        n = 5
        for _, fs in self.terms:
            n += 1
            for f in fs:
                kind = self.transform_of(f)[0]
                n += 1 if kind == 1 else (self.D if kind == 2 else 0)
                n += 1 if f["p"] is not None else 0
                n += self.D if f["r"] is not None else 0
        return n

    def params_grad(self, g):
        """chain rule from the descriptor gradient g (agp_post_logpdf_grad layout) to kernel_params order: every copy that
        flattening made of a parameter contributes; no division by a parameter's value"""
        D = self.D
        out = [np.zeros_like(np.asarray(v, dtype=np.float64)) if np.ndim(v) else 0.0 for v in self.vals]

        def add(i, x):
            if np.ndim(self.vals[i]) == 0:
                out[i] = out[i] + float(np.sum(x))
            elif self.vals[i].shape[0] == 1 and D > 1:
                out[i] = out[i] + np.array([np.sum(x)])
            else:
                out[i] = out[i] + x
        pos = 5
        for s_, fs in self.terms:
            for j, i in enumerate(s_):
                add(i, g[pos] * _prod_except(self.vals, s_, j))
            pos += 1
            for f in fs:
                kind = self.transform_of(f)[0]
                if kind == 1:
                    for j, i in enumerate(f["tr"]):
                        add(i, g[pos] * _prod_except(self.vals, f["tr"], j))
                    pos += 1
                elif kind == 2:
                    gv = np.asarray(g[pos:pos + D])
                    for j, i in enumerate(f["tr"]):
                        add(i, gv * _prod_except(self.vals, f["tr"], j, D))
                    pos += D
                if f["p"] is not None:
                    add(f["p"], g[pos])
                    pos += 1
                if f["r"] is not None:
                    add(f["r"], np.asarray(g[pos:pos + D]))
                    pos += D
        return out


def _composite_diag(k: Kernel, a):
    """kernelmatrix_diag of a composite kernel: sum_t v_t prod_f kappa_f(x, x) -- 1 for stationary, RQ, Periodic and
    White factors, c for Constant, |x~|^2 + c for Linear (like the single-kernel Linear diagonal, formed host-side)"""
    fl = _Flat(k, a.shape[1])
    out = np.zeros(a.shape[0], dtype=a.dtype)
    for s_, fs in fl.terms:
        t = np.full(a.shape[0], _prod_except(fl.vals, s_, -1), dtype=a.dtype)
        for f in fs:
            if f["family"] == CONSTANT:
                t = t * a.dtype.type(fl.vals[f["p"]])
            elif f["family"] == LINEAR:
                kind, s, v = fl.transform_of(f)
                xt = a * (a.dtype.type(s) if v is None else v.astype(a.dtype))
                t = t * ((xt * xt).sum(1) + a.dtype.type(fl.vals[f["p"]]))
        out = out + t
    return out


def kernel_params(k: Kernel):
    """Depth-first list of every parameter of a kernel tree: each ScaledKernel sigma^2 (or variance other than 1), each
    transform's s / v, and RQ
    alpha, Periodic r, Linear c and Constant c -- the order of logpdf_grad(...)["kernel"] for a composite kernel."""
    vals = []
    _walk(k, vals)
    return vals


def with_kernel_params(k: Kernel, vals):
    """The same tree with its parameters replaced, in kernel_params(k) order."""
    it = iter(list(vals))

    def rebuild(k):
        variance = float(next(it)) if (k.scaled or k.variance != 1.0) else k.variance
        t = k.transform
        if t is not None:
            v = next(it)
            t = ScaleTransform(float(v)) if isinstance(t, ScaleTransform) else ARDTransform(v)
        if isinstance(k, _CompositeKernel):
            out = k._copy(variance=variance)
            out.transform = t
            out.kernels = [rebuild(ch) for ch in k.kernels]
            return out
        out = k._copy(variance=variance)
        out.transform = t
        if k.family == RQ:
            out.alpha = float(next(it))
        elif k.family in (LINEAR, CONSTANT):
            out.c = float(next(it))
        if k.family == PERIODIC:
            out.r = np.ascontiguousarray(next(it), dtype=np.float64).ravel()
        return out
    return rebuild(k)


class ColVecs:
    """ColVecs(X): X is D x N, each COLUMN a point (KernelFunctions.ColVecs)."""

    def __init__(self, X):
        X = np.asarray(X)
        assert X.ndim == 2
        self.X = X

    def __len__(self):
        return self.X.shape[1]


class RowVecs:
    """RowVecs(X): X is N x D, each ROW a point (KernelFunctions.RowVecs)."""

    def __init__(self, X):
        X = np.asarray(X)
        assert X.ndim == 2
        self.X = X

    def __len__(self):
        return self.X.shape[0]


class _Points:
    """Engine view of an input collection: a C-contiguous [n, D] host array == D x N column-major
    == AGP_POINT_MAJOR for the ABI (so both wrappers cost at most one host transpose)."""

    def __init__(self, x):
        if isinstance(x, _Points):
            self.a = x.a
        elif isinstance(x, ColVecs):
            self.a = np.ascontiguousarray(x.X.T)
        elif isinstance(x, RowVecs):
            self.a = np.ascontiguousarray(x.X)
        else:
            v = np.asarray(x)
            if v.ndim != 1:
                raise TypeError("inputs must be a vector of reals, ColVecs(X) or RowVecs(X)")
            self.a = np.ascontiguousarray(v.reshape(-1, 1))
        if self.a.dtype not in (np.float32, np.float64):
            self.a = self.a.astype(np.float64)
        self.n, self.D = self.a.shape

    def astype(self, dt):
        p = _Points.__new__(_Points)
        p.a = np.ascontiguousarray(self.a, dtype=dt)
        p.n, p.D = self.n, self.D
        return p

    def julia_items(self):
        """what `map(f, x)` would iterate over (src/mean_function.jl:52-55)."""
        return self.a[:, 0] if self.D == 1 else self.a


def vcat(x, y):
    return _Points_from(np.concatenate([_Points(x).a, _Points(y).a], 0))


def _Points_from(a):
    p = _Points.__new__(_Points)
    p.a = np.ascontiguousarray(a)
    p.n, p.D = p.a.shape
    return p


# ---------------------------------------------------------------------------------------------
# mean functions (src/mean_function.jl)
# ---------------------------------------------------------------------------------------------
class MeanFunction:
    pass


class ZeroMean(MeanFunction):
    def vector(self, pts, dt):
        return np.zeros(pts.n, dtype=dt)

    def spec(self, pts, dt):
        return 0, 0.0, None


class ConstMean(MeanFunction):
    def __init__(self, c):
        self.c = float(c)

    def vector(self, pts, dt):
        return np.full(pts.n, self.c, dtype=dt)

    def spec(self, pts, dt):
        return 1, self.c, None


class CustomMean(MeanFunction):
    """arbitrary host closure: evaluated host-side and shipped as a vector (SURVEY s8a row 2)."""

    def __init__(self, f):
        self.f = f

    def vector(self, pts, dt):
        return np.array([self.f(xi) for xi in pts.julia_items()], dtype=dt)

    def spec(self, pts, dt):
        return 2, 0.0, self.vector(pts, dt)


# ---------------------------------------------------------------------------------------------
# engine singleton
# ---------------------------------------------------------------------------------------------
class Engine:
    def __init__(self, device: Optional[int] = None):
        L = cabi.lib()
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", "0"))
        h = C.c_void_p()
        rc = L.agp_init(C.byref(h), device, None)
        if rc != cabi.AGP_OK:
            raise AGPError(rc, "agp_init failed on device %d (no CUDA device? there is no CPU fallback)" % device)
        self.L, self.h, self.device = L, h, device

    def check(self, rc):
        if rc == cabi.AGP_OK:
            return
        msg = self.L.agp_last_error(self.h).decode()
        if rc == cabi.AGP_ERR_NOT_POSDEF:
            raise PosDefException(int(self.L.agp_last_info(self.h)), msg)
        if rc == cabi.AGP_ERR_DIM_MISMATCH:
            raise DimensionMismatch(msg)
        raise AGPError(rc, msg)

    def timings(self):
        buf = (C.c_double * 8)()
        n = self.L.agp_last_timings(self.h, buf, 8)
        keys = ["total", "h2d", "gram", "cholesky", "solves", "d2h", "predict", "trailing"]
        return {k: buf[i] for i, k in enumerate(keys[:n])}

    def launch_count(self):
        return int(self.L.agp_launch_count(self.h))

    def set_memspace(self, m):
        self.check(self.L.agp_set_memspace(self.h, m))

    def get_config(self):
        c = cabi.agp_config()
        self.check(self.L.agp_get_config(self.h, C.byref(c)))
        return c

    def set_config(self, **kw):
        """tile_nb / fp64_mode / lookahead / ozaki_slices of the live context"""
        c = self.get_config()
        for k_, v in kw.items():
            setattr(c, k_, v)
        self.check(self.L.agp_set_config(self.h, C.byref(c)))


_engine = None


def engine() -> Engine:
    global _engine
    if _engine is None:
        _engine = Engine()
    return _engine


def _kernel_struct(k: Kernel, dt, keep, D=None):
    if isinstance(k, _CompositeKernel) or k.family > LINEAR:
        if not isinstance(k, _CompositeKernel):  # a lone RQ / Periodic / White / Constant is a one-factor composite
            k = KernelSum(k)
        return _Flat(k, D).struct(dt, keep)
    ks = cabi.agp_kernel()
    ks.family, ks.variance, ks.linear_c, ks.scale = k.family, k.variance, k.c, 1.0
    t = k.transform
    if t is None:
        ks.transform = 0
    elif isinstance(t, ScaleTransform):
        ks.transform, ks.scale = 1, t.s
    else:
        v = np.ascontiguousarray(t.v, dtype=dt)
        keep.append(v)
        ks.transform, ks.ard = 2, v.ctypes.data
    return ks


def _mean_struct(spec, keep):
    kind, c, v = spec
    ms = cabi.agp_mean()
    ms.kind, ms.c = kind, c
    if v is not None:
        keep.append(v)
        ms.v = v.ctypes.data
    return ms


def _noise_struct(s2, n, dt, keep):
    ns = cabi.agp_noise()
    if np.ndim(s2) == 0:
        ns.kind, ns.s = 0, float(s2)
    else:
        v = np.ascontiguousarray(s2, dtype=dt).ravel()
        if v.shape[0] != n:
            raise DimensionMismatch("noise vector has length %d, expected %d" % (v.shape[0], n))
        keep.append(v)
        ns.kind, ns.v = 1, v.ctypes.data
    return ns


def _vfe_mean_cov(p: "ApproxPosteriorGP", pts: _Points):
    """mean_and_cov(::ApproxPosteriorGP, x*) (src/sparse_approximations.jl:205-210) through agp_vfe_mean_cov (EXPERIMENTAL)."""
    eng = engine()
    pts = pts.astype(p.dtype)
    m = np.empty(pts.n, dtype=p.dtype)
    Cv = np.empty((pts.n, pts.n), dtype=p.dtype, order="F")
    eng.check(eng.L.agp_vfe_mean_cov(p.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, cabi.ptr(m), cabi.ptr(Cv)))
    if isinstance(p.prior.mean, CustomMean):
        m = m + p.prior.mean.vector(pts, p.dtype)
    return m, Cv


def _vfe_post_logpdf(fx: "FiniteGP", y):
    """logpdf(f_approx_post(x*, s2), y) on the device (agp_vfe_post_logpdf, EXPERIMENTAL)."""
    eng = engine()
    p = fx.f
    dt = p.dtype
    pts = fx.x.astype(dt)
    Y = np.asarray(y, dtype=dt)
    vec = Y.ndim == 1
    Yf = Y.reshape(-1, 1) if vec else Y
    if Yf.shape[0] != pts.n:
        raise DimensionMismatch("length(fx) = %d but y has %d rows" % (pts.n, Yf.shape[0]))
    if isinstance(p.prior.mean, CustomMean):  # the handle knows Zero/Const means: a closure mean is removed here
        Yf = Yf - p.prior.mean.vector(pts, dt)[:, None]
    keep = []
    ns = _noise_struct(fx.s2, pts.n, dt, keep)
    lp = np.empty(Yf.shape[1], dtype=dt)
    for s0 in range(0, Yf.shape[1], 128):
        s1 = min(Yf.shape[1], s0 + 128)
        Yc = np.asfortranarray(Yf[:, s0:s1])
        eng.check(eng.L.agp_vfe_post_logpdf(p.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, C.byref(ns), cabi.ptr(Yc),
                                            s1 - s0, cabi.ptr(lp[s0:s1])))
    return lp[0] if vec else lp


def _vfe_post_rand_from_normals(fx: "FiniteGP", Z, squeeze=False):
    eng = engine()
    p = fx.f
    dt = p.dtype
    pts = fx.x.astype(dt)
    Z = np.asfortranarray(np.asarray(Z, dtype=dt).reshape(pts.n, -1))
    keep = []
    ns = _noise_struct(fx.s2, pts.n, dt, keep)
    out = np.empty_like(Z, order="F")
    eng.check(eng.L.agp_vfe_post_rand(p.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, C.byref(ns), cabi.ptr(Z), Z.shape[1],
                                      cabi.ptr(out)))
    if isinstance(p.prior.mean, CustomMean):
        out = out + p.prior.mean.vector(pts, dt)[:, None]
    return out[:, 0] if squeeze else out


# ---------------------------------------------------------------------------------------------
# GP / FiniteGP / PosteriorGP  (src/base_gp.jl, src/finite_gp_projection.jl, src/exact_gpr_posterior.jl)
# ---------------------------------------------------------------------------------------------
default_s2 = 1e-18  # src/finite_gp_projection.jl:17


class AbstractGP:
    def __call__(self, x, s2=default_s2, obsdim=None):
        """(f::AbstractGP)(x...) src/finite_gp_projection.jl:32; (f)(X::AbstractMatrix, args...; obsdim) :33-37 --
        obsdim = 1: rows are points (RowVecs), obsdim = 2: columns are points (ColVecs); a bare matrix without obsdim
        is ambiguous (the reference deprecated its default) and is rejected."""
        if obsdim is not None:
            X = np.asarray(x)
            if X.ndim != 2 or obsdim not in (1, 2):
                raise TypeError("obsdim applies to a matrix of inputs and is 1 (rows) or 2 (columns)")
            x = RowVecs(X) if obsdim == 1 else ColVecs(X)
        return FiniteGP(self, x, s2)


class GP(AbstractGP):
    """GP(kernel) / GP(mean, kernel) / GP(c::Real, kernel)  (src/base_gp.jl:57-64)."""

    def __init__(self, *args):
        if len(args) == 1:
            mean, kernel = ZeroMean(), args[0]
        else:
            mean, kernel = args
            if isinstance(mean, (int, float, np.integer, np.floating)):  # GP(c::Real, kernel), src/base_gp.jl:64
                mean = ConstMean(mean)
            elif not isinstance(mean, MeanFunction):
                mean = CustomMean(mean)
        if not isinstance(kernel, Kernel):
            raise TypeError("kernel must be one of the device-supported KernelFunctions kernels")
        self.mean, self.kernel = mean, kernel


class FiniteGP:
    """FiniteGP(f, x, Sigma_y) (src/finite_gp_projection.jl:7-21): scalar s2 -> Fill, vector -> Diagonal."""

    def __init__(self, f, x, s2=default_s2):
        self.f, self.x = f, _Points(x)
        # the container the inputs came in, for gradients shaped like it: ColVecs, RowVecs (or a point set) or a vector
        self.x_kind = "col" if isinstance(x, ColVecs) else ("row" if isinstance(x, (RowVecs, _Points)) else "vec")
        if np.ndim(s2) == 2:
            raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "dense Sigma_y is outside the device hot path (SURVEY s8a)")
        self.s2 = s2
        self.dtype = np.result_type(self.x.a.dtype, np.float32)

    def __len__(self):
        return self.x.n

    @property
    def Sigma_y_diag(self):
        return np.full(self.x.n, self.s2, dtype=self.dtype) if np.ndim(self.s2) == 0 else np.asarray(self.s2, self.dtype)


DeviceData = namedtuple("DeviceData", "alpha C x delta")


class DeviceCholesky:
    """The `C` field of PosteriorGP.data: a handle to the device-resident factor (boundary #2,
    src/util/common_covmat_ops.jl).  `.U` exports the upper factor like `C.U` in the reference."""

    def __init__(self, eng: Engine, handle, dtype):
        self.eng, self.h, self.dtype = eng, handle, dtype

    def __del__(self):
        try:
            if self.h:
                self.eng.L.agp_post_free(self.h)
                self.h = None
        except Exception:
            pass

    @property
    def n(self):
        return int(self.eng.L.agp_post_n(self.h))

    @property
    def U(self):
        out = np.empty((self.n, self.n), dtype=self.dtype, order="F")
        self.eng.check(self.eng.L.agp_post_factor_export(self.h, cabi.ptr(out)))
        return out

    def logdet(self):
        v = C.c_double()
        self.eng.check(self.eng.L.agp_post_logdet(self.h, C.byref(v)))
        return v.value

    def solve_lower(self, B):
        """U' \\ B"""
        B = np.asarray(B, dtype=self.dtype)
        vec = B.ndim == 1
        Bf = np.asfortranarray(B.reshape(self.n, -1))
        out = np.empty_like(Bf, order="F")
        self.eng.check(self.eng.L.agp_post_solve_lower(self.h, cabi.ptr(Bf), Bf.shape[1], cabi.ptr(out)))
        return out[:, 0] if vec else out


# the operator API of src/util/common_covmat_ops.jl on a device factor
def Xt_invA_X(A: DeviceCholesky, X):  # :54-58
    V = A.solve_lower(X)
    return float(np.sum(V * V)) if V.ndim == 1 else V.T @ V


def Xt_invA_Y(X, A: DeviceCholesky, Y):  # :60
    return A.solve_lower(X).T @ A.solve_lower(Y)


def diag_Xt_invA_X(A: DeviceCholesky, X):  # :90
    V = A.solve_lower(X)
    return np.array([np.sum(V * V)]) if V.ndim == 1 else np.sum(V * V, axis=0)


def tr_Xt_invA_X(A: DeviceCholesky, X):  # :101
    V = A.solve_lower(X)
    return float(np.sum(V * V))


class PosteriorGP(AbstractGP):
    """PosteriorGP(prior, data=(alpha, C, x, delta)) (src/exact_gpr_posterior.jl:1-4)."""

    def __init__(self, prior, data):
        self.prior, self.data = prior, data


def _prior_of(fx: FiniteGP) -> GP:
    f = fx.f
    if not isinstance(f, GP):
        raise TypeError("expected a FiniteGP over a prior GP")
    return f


def _fit(fx: FiniteGP, Y, want_post: bool, want_alpha: bool):
    eng = engine()
    f = _prior_of(fx)
    dt = fx.dtype
    pts = fx.x.astype(dt)
    Y = np.asarray(Y)
    vec = Y.ndim == 1
    Yf = np.asfortranarray(Y.reshape(-1, 1) if vec else Y, dtype=dt)
    if Yf.shape[0] != pts.n:
        raise DimensionMismatch("length(fx) = %d but Y has %d rows" % (pts.n, Yf.shape[0]))
    S = Yf.shape[1]
    keep = []
    ks = _kernel_struct(f.kernel, dt, keep, D=pts.D)
    ms = _mean_struct(f.mean.spec(pts, dt), keep)
    ns = _noise_struct(fx.s2, pts.n, dt, keep)
    lp = np.empty(S, dtype=dt)
    alpha = np.empty(pts.n, dtype=dt) if want_alpha else None
    post = C.c_void_p()
    # one call whatever S is: the library carries 128 columns through the factorisation and solves the rest against the
    # same factor (ONE Gram + ONE Cholesky)
    rc = eng.L.agp_fit(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), cabi.AGP_POINT_MAJOR,
                       cabi.ptr(pts.a), pts.n, pts.D, cabi.ptr(Yf), S, cabi.ptr(lp),
                       cabi.ptr(alpha) if want_alpha else None, C.byref(post) if want_post else None)
    eng.check(rc)
    lpv = lp[0] if vec else lp
    if not want_post:
        return lpv, None
    delta = Yf[:, 0] - f.mean.vector(pts, dt)
    data = DeviceData(alpha=alpha, C=DeviceCholesky(eng, post, dt), x=fx.x, delta=delta)
    p = PosteriorGP(f, data)
    p.fx = fx  # the FiniteGP it was conditioned on: its noise and input container shape the posterior's gradients
    return lpv, p


def logpdf(fx: FiniteGP, y):
    """logpdf(fx, y) (src/finite_gp_projection.jl:306-311); matrix y -> per-column values."""
    if isinstance(fx.f, PosteriorGP):
        return _post_logpdf(fx, y)
    if isinstance(fx.f, ApproxPosteriorGP):
        return _vfe_post_logpdf(fx, y)
    if not isinstance(fx.f, GP):
        raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "logpdf of a FiniteGP over %s is outside the device hot path"
                       % type(fx.f).__name__)
    return _fit(fx, y, False, False)[0]


def _post_args(fx: FiniteGP):
    p: PosteriorGP = fx.f
    dt = p.data.C.dtype
    pts = fx.x.astype(dt)
    if pts.D != p.data.x.D:
        raise DimensionMismatch("test points have D=%d, training points D=%d" % (pts.D, p.data.x.D))
    keep = []
    ms = _mean_struct(p.prior.mean.spec(pts, dt), keep)
    ns = _noise_struct(fx.s2, pts.n, dt, keep)
    return p, dt, pts, ms, ns, keep


def _post_logpdf(fx: FiniteGP, y):
    """logpdf(f_post(x*, s2), y) (src/finite_gp_projection.jl:306-318 over src/exact_gpr_posterior.jl:78-83):
    posterior covariance, noise add, Cholesky and the quadratic form all on the device (agp_post_logpdf)."""
    eng = engine()
    p, dt, pts, ms, ns, keep = _post_args(fx)
    Y = np.asarray(y, dtype=dt)
    vec = Y.ndim == 1
    Yf = Y.reshape(-1, 1) if vec else Y
    if Yf.shape[0] != pts.n:
        raise DimensionMismatch("length(fx) = %d but y has %d rows" % (pts.n, Yf.shape[0]))
    S = Yf.shape[1]
    lp = np.empty(S, dtype=dt)
    for s0 in range(0, S, 128):
        s1 = min(S, s0 + 128)
        Yc = np.asfortranarray(Yf[:, s0:s1])
        eng.check(eng.L.agp_post_logpdf(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, C.byref(ms),
                                        C.byref(ns), cabi.ptr(Yc), s1 - s0, cabi.ptr(lp[s0:s1])))
    return lp[0] if vec else lp


def _post_rand_from_normals(fx: FiniteGP, Z, squeeze=False):
    """rand(f_post(x*, s2), S) (src/finite_gp_projection.jl:233-240) through agp_post_rand."""
    eng = engine()
    p, dt, pts, ms, ns, keep = _post_args(fx)
    Z = np.asfortranarray(np.asarray(Z, dtype=dt).reshape(pts.n, -1))
    out = np.empty_like(Z, order="F")
    eng.check(eng.L.agp_post_rand(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, C.byref(ms), C.byref(ns),
                                  cabi.ptr(Z), Z.shape[1], cabi.ptr(out)))
    return out[:, 0] if squeeze else out


def loglikelihood(fx: FiniteGP, Y):  # src/finite_gp_projection.jl:304
    return np.sum(logpdf(fx, Y))


def posterior(fx, y=None, *rest):
    """posterior(fx, y) (src/exact_gpr_posterior.jl:29-35); posterior(vfe, fx, y) (src/sparse_approximations.jl:58-75);
    posterior(fx::FiniteGP{<:PosteriorGP}, y) sequential conditioning (src/exact_gpr_posterior.jl:46-56)."""
    if isinstance(fx, VFE):
        return _vfe_posterior(fx, y, rest[0])
    if isinstance(fx.f, PosteriorGP):
        return _posterior_sequential(fx, y)
    return _fit(fx, y, True, True)[1]


def fit(fx: FiniteGP, y):
    """Fused logpdf + posterior from ONE Gram and ONE factorisation (the reference does two:
    src/finite_gp_projection.jl:307-308 and src/exact_gpr_posterior.jl:30-31)."""
    return _fit(fx, y, True, True)


def _grad_buffer(k: Kernel, D, h=None):
    """(g, flat): the zeroed gradient vector for kernel k and, for a composite, the _Flat that maps it back onto
    kernel_params(k) (None otherwise).  With a posterior handle h a composite's length is the handle's."""
    if not (isinstance(k, _CompositeKernel) or k.family > LINEAR):
        return np.zeros(5 + D, dtype=np.float64), None
    flat = _Flat(k if isinstance(k, _CompositeKernel) else KernelSum(k), D)
    n = int(engine().L.agp_post_grad_len(h)) if h is not None else flat.grad_len()
    return np.zeros(n, dtype=np.float64), flat


def _grad_result(g, flat, k: Kernel, D, mean: "MeanFunction", noise, mean_v):
    """The gradient dict's kernel, noise and mean keys from g: "kernel" (composite) or "variance", "scale" | "ard",
    "linear_c"; "noise" (the per-point vector `noise`, else g[3]); "mean_c" (ConstMean) or "mean_v" (CustomMean)."""
    if flat is not None:
        res = {"kernel": flat.params_grad(g)}
    else:
        res = {"variance": g[0]}
        if isinstance(k.transform, ScaleTransform):
            res["scale"] = g[1]
        elif isinstance(k.transform, ARDTransform):
            res["ard"] = g[5:5 + D].copy()
        if k.family == LINEAR:
            res["linear_c"] = g[2]
    res["noise"] = g[3] if noise is None else noise.astype(np.float64)
    if isinstance(mean, ConstMean):
        res["mean_c"] = g[4]
    elif isinstance(mean, CustomMean):
        res["mean_v"] = mean_v.astype(np.float64)
    return res


def _points_grad(kind, n, D, dt):
    """The buffer a point-major input gradient of n points comes back in, shaped like the container kind: D x n
    column-major (ColVecs), length n (a vector), or n x D row-major (RowVecs) -- all the same memory order."""
    return {"col": lambda: np.empty((D, n), dtype=dt, order="F"), "vec": lambda: np.empty(n, dtype=dt),
            "row": lambda: np.empty((n, D), dtype=dt)}[kind]()


def _cols_and_weights(Y, lp_bar, n, dt):
    """(ndim of Y, Y as an n x S Fortran array, S, lp_bar as float64 or None for all ones)"""
    Yin = np.asarray(Y)
    Yf = np.asfortranarray(Yin.reshape(-1, 1) if Yin.ndim == 1 else Yin, dtype=dt)
    if Yf.shape[0] != n:
        raise DimensionMismatch("length(fx) = %d but Y has %d rows" % (n, Yf.shape[0]))
    S = Yf.shape[1]
    w = None if lp_bar is None else np.ascontiguousarray(lp_bar, dtype=np.float64).ravel()
    if w is not None and w.shape[0] != S:
        raise DimensionMismatch("lp_bar has %d entries, Y has %d columns" % (w.shape[0], S))
    return Yin.ndim, Yf, S, w


def logpdf_grad(fx: FiniteGP, y, inputs=False):
    """EXPERIMENTAL (device path not yet validated): (logpdf, gradient dict) of logpdf(fx, y) w.r.t. the kernel variance,
    ScaleTransform s / ARDTransform v, LinearKernel c, the noise (scalar or per-point) and the mean (constant or vector)
    -- the cotangents Zygote returns through the reference (test/finite_gp_projection.jl:152-178).  One fit, then
    agp_post_logpdf_grad on its factor.

    inputs=True also returns out["x"], the gradient with respect to the input points, shaped like the container fx was
    built from (RowVecs: N x D, ColVecs: D x N, a vector: length N) in the handle's dtype; both come from one
    agp_post_logpdf_grad_x call.  A CustomMean is treated as a constant of x."""
    lp, post = _fit(fx, y, True, True)
    eng = engine()
    f = post.prior
    dt = post.data.C.dtype
    D = post.data.x.D
    k = f.kernel
    g, flat = _grad_buffer(k, D, post.data.C.h)
    per_point = np.ndim(fx.s2) != 0
    nd = np.empty(len(fx), dtype=dt) if (per_point or isinstance(f.mean, CustomMean)) else None
    if inputs:
        # a RowVecs gradient comes back feature-major, N x D column-major like the other containers' memory
        xk = fx.x_kind
        layout = cabi.AGP_FEATURE_MAJOR if xk == "row" else cabi.AGP_POINT_MAJOR
        xg = np.empty((len(fx), D), dtype=dt, order="F") if xk == "row" else _points_grad(xk, len(fx), D, dt)
        eng.check(eng.L.agp_post_logpdf_grad_x(post.data.C.h, g.ctypes.data_as(C.POINTER(C.c_double)), cabi.ptr(nd), layout,
                                               cabi.ptr(xg)))
    else:
        eng.check(eng.L.agp_post_logpdf_grad(post.data.C.h, g.ctypes.data_as(C.POINTER(C.c_double)), cabi.ptr(nd)))
    # composite: out["kernel"][i] is the derivative in kernel_params(k)[i] (the descriptor's gradient mapped back)
    out = _grad_result(g, flat, k, D, f.mean, nd if per_point else None, post.data.alpha)
    if inputs:
        out["x"] = xg
    return lp, out


def loglikelihood_grad(fx: FiniteGP, Y, lp_bar=None, inputs=False):
    """(logpdf vector, gradient dict) of sum_s lp_bar[s] * logpdf(fx, Y[:, s]) for a matrix Y (N x S, or a vector as one
    column) over a prior GP -- what Zygote returns through the reference's logpdf(fx, Y::AbstractMatrix) and
    loglikelihood(fx, Y) (test/finite_gp_projection.jl:165-178).  lp_bar=None is all ones: the gradient of
    loglikelihood(fx, Y).  One fit and one agp_post_logpdf_grad_cols call whatever S is (one factorisation, one C^-1).
    The dict has the keys of logpdf_grad ("kernel" for a composite, else "variance", "scale" | "ard", "linear_c"; "noise"
    scalar or per-point; "mean_c" | "mean_v") and "Y", the cotangent of Y, shaped like Y.  inputs=True also returns
    out["x"], the gradient with respect to the input points, shaped like the container fx was built from (RowVecs: N x D,
    ColVecs: D x N, a vector: length N).  A CustomMean is treated as a constant of x: the caller chains through
    out["mean_v"]."""
    if not isinstance(fx.f, GP):
        raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "the gradient of logpdf over a matrix Y is implemented for a FiniteGP over "
                       "a prior GP, not over %s" % type(fx.f).__name__)
    dt = fx.dtype
    pts = fx.x.astype(dt)
    N, D = pts.n, pts.D
    ndim, Yf, S, w = _cols_and_weights(Y, lp_bar, N, dt)
    lp, post = _fit(fx, Yf, True, False)
    eng = engine()
    f = fx.f
    k = f.kernel
    g, flat = _grad_buffer(k, D)
    nd = np.empty(N, dtype=dt) if np.ndim(fx.s2) != 0 else None
    md = np.empty(N, dtype=dt) if isinstance(f.mean, CustomMean) else None
    yb = np.empty((N, S), dtype=dt, order="F")
    xg = _points_grad(fx.x_kind, N, D, dt) if inputs else None  # the points go in point-major
    keep = []
    ms = _mean_struct(f.mean.spec(pts, dt), keep)
    eng.check(eng.L.agp_post_logpdf_grad_cols(post.data.C.h, C.byref(ms), cabi.ptr(Yf), S,
                                              None if w is None else w.ctypes.data_as(C.POINTER(C.c_double)),
                                              g.ctypes.data_as(C.POINTER(C.c_double)), cabi.ptr(nd), cabi.ptr(md),
                                              cabi.AGP_POINT_MAJOR, cabi.ptr(xg), cabi.ptr(yb)))
    res = _grad_result(g, flat, k, D, f.mean, nd, md)
    res["Y"] = yb[:, 0].copy() if ndim == 1 else yb
    if inputs:
        res["x"] = xg
    return np.atleast_1d(lp), res


def posterior_logpdf_grad(fx: FiniteGP, Y, lp_bar=None, inputs=False):
    """(logpdf, gradient dict) of sum_s lp_bar[s] * logpdf(fx, Y[:, s]) for fx = p(x*, s2*) over an exact posterior
    p = posterior(fx0, y): the held-out log-likelihood logpdf(posterior(fx0, y)(x*, s2*), y*) differentiated with respect
    to both the training and the test side, in one agp_post_pred_logpdf_grad call on p's handle.  Y is M x S (or a vector
    as one column); lp_bar=None is all ones.  The dict has the kernel keys of logpdf_grad ("kernel" for a composite, else
    "variance", "scale" | "ard", "linear_c"), the training side "noise" (scalar or per-point, as fx0's noise), "mean_c"
    (ConstMean) or "mean_v" (CustomMean, at x) and "y" (the cotangent of y); the test side "noise_s" (scalar or per-point,
    as fx's noise), "mean_s_v" (CustomMean, at x*) and "Y" (shaped like Y).  A ConstMean's "mean_c" counts both sides.
    inputs=True also returns "x" and "xs", the gradients with respect to the training and the test inputs, shaped like the
    containers they came in (RowVecs: N x D, ColVecs: D x N, a vector: length N).  A CustomMean is treated as a constant
    of the inputs.  Only a posterior straight from posterior(fx0, y) is supported (not a sequentially conditioned one)."""
    p = fx.f
    if not isinstance(p, PosteriorGP) or getattr(p, "fx", None) is None:
        raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "the gradient of the held-out logpdf needs a FiniteGP over posterior(fx, y), "
                       "not over %s" % type(p).__name__)
    eng = engine()
    p, dt, pts, ms, ns, keep = _post_args(fx)
    fx0 = p.fx
    N, M, D = p.data.x.n, pts.n, pts.D
    ndim, Yf, S, w = _cols_and_weights(Y, lp_bar, M, dt)
    f = p.prior
    k = f.kernel
    g, flat = _grad_buffer(k, D, p.data.C.h)
    lp = np.empty(S, dtype=dt)
    nd = np.empty(N, dtype=dt) if np.ndim(fx0.s2) != 0 else None
    md = np.empty(N, dtype=dt) if isinstance(f.mean, CustomMean) else None
    yb = np.empty(N, dtype=dt)
    nsd = np.empty(M, dtype=dt)
    msd = np.empty(M, dtype=dt) if isinstance(f.mean, CustomMean) else None
    ysb = np.empty((M, S), dtype=dt, order="F")
    xg = _points_grad(fx0.x_kind, N, D, dt) if inputs else None  # the points go in point-major
    xsg = _points_grad(fx.x_kind, M, D, dt) if inputs else None
    dbl = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))
    eng.check(eng.L.agp_post_pred_logpdf_grad(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), M, C.byref(ms), C.byref(ns),
                                              cabi.ptr(Yf), S, dbl(w), cabi.ptr(lp), dbl(g), cabi.ptr(nd), cabi.ptr(md),
                                              cabi.ptr(yb), cabi.ptr(xg), cabi.ptr(nsd), cabi.ptr(msd), cabi.ptr(ysb),
                                              cabi.ptr(xsg)))
    res = _grad_result(g, flat, k, D, f.mean, nd, md)
    res["y"] = yb
    res["noise_s"] = nsd.astype(np.float64) if np.ndim(fx.s2) != 0 else float(np.sum(nsd, dtype=np.float64))
    if msd is not None:
        res["mean_s_v"] = msd.astype(np.float64)
    res["Y"] = ysb[:, 0].copy() if ndim == 1 else ysb
    if inputs:
        res["x"], res["xs"] = xg, xsg
    return (lp[0] if ndim == 1 else lp), res


def posterior_rand_grad(fx: FiniteGP, Z, out_bar, inputs=False):
    """(out, gradient dict) of the posterior samples out = rand(fx, S) = mu* + L* Z at the caller's standard normals Z,
    pulled back from the cotangent out_bar, for fx = p(x*, s2*) over an exact posterior p = posterior(fx0, y): what
    Zygote returns through rand over a posterior, for Monte Carlo acquisition functions and losses built on
    reparameterised samples.  One agp_post_rand_grad call on p's handle; out is agp_post_rand's at the same Z.  Z and
    out_bar are M x S (or vectors as one column).  The dict has the keys of posterior_logpdf_grad with "Z" (the cotangent
    of the normals, shaped like Z) in place of "Y": the kernel keys, the training side "noise", "mean_c" | "mean_v" and
    "y", the test side "noise_s" and "mean_s_v"; a ConstMean's "mean_c" counts both sides.  inputs=True also returns
    "x" and "xs", shaped like the containers the points came in.  A CustomMean is treated as a constant of the inputs.
    Only a posterior straight from posterior(fx0, y) is supported (not a sequentially conditioned one)."""
    p = fx.f
    if not isinstance(p, PosteriorGP) or getattr(p, "fx", None) is None:
        raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "the gradient of rand over a posterior needs a FiniteGP over "
                       "posterior(fx, y), not over %s" % type(p).__name__)
    eng = engine()
    p, dt, pts, ms, ns, keep = _post_args(fx)
    fx0 = p.fx
    N, M, D = p.data.x.n, pts.n, pts.D
    ndim, Zf, S, _ = _cols_and_weights(Z, None, M, dt)
    _, Ob, _, _ = _cols_and_weights(out_bar, None, M, dt)
    if Ob.shape != Zf.shape:
        raise DimensionMismatch("out_bar has shape %s, Z has %s" % (Ob.shape, Zf.shape))
    f = p.prior
    k = f.kernel
    g, flat = _grad_buffer(k, D, p.data.C.h)
    out = np.empty((M, S), dtype=dt, order="F")
    eng.check(eng.L.agp_post_rand(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), M, C.byref(ms), C.byref(ns),
                                  cabi.ptr(Zf), S, cabi.ptr(out)))
    nd = np.empty(N, dtype=dt) if np.ndim(fx0.s2) != 0 else None
    md = np.empty(N, dtype=dt) if isinstance(f.mean, CustomMean) else None
    yb = np.empty(N, dtype=dt)
    nsd = np.empty(M, dtype=dt)
    msd = np.empty(M, dtype=dt) if isinstance(f.mean, CustomMean) else None
    zb = np.empty((M, S), dtype=dt, order="F")
    xg = _points_grad(fx0.x_kind, N, D, dt) if inputs else None  # the points go in point-major
    xsg = _points_grad(fx.x_kind, M, D, dt) if inputs else None
    eng.check(eng.L.agp_post_rand_grad(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), M, C.byref(ms), C.byref(ns),
                                       cabi.ptr(Zf), S, cabi.ptr(Ob), g.ctypes.data_as(C.POINTER(C.c_double)),
                                       cabi.ptr(nd), cabi.ptr(md), cabi.ptr(yb), cabi.ptr(xg), cabi.ptr(nsd),
                                       cabi.ptr(msd), cabi.ptr(zb), cabi.ptr(xsg)))
    res = _grad_result(g, flat, k, D, f.mean, nd, md)
    res["y"] = yb
    res["noise_s"] = nsd.astype(np.float64) if np.ndim(fx.s2) != 0 else float(np.sum(nsd, dtype=np.float64))
    if msd is not None:
        res["mean_s_v"] = msd.astype(np.float64)
    res["Z"] = zb[:, 0].copy() if ndim == 1 else zb
    if inputs:
        res["x"], res["xs"] = xg, xsg
    return (out[:, 0].copy() if ndim == 1 else out), res


def posterior_mean_var_grad(fx: FiniteGP, mean_bar, var_bar, inputs=False, training=True):
    """((mean, var), gradient dict) of mean_and_var(fx) for fx = p(x*, s2*) over an exact posterior p = posterior(fx0, y),
    pulled back from the cotangents mean_bar and var_bar (M values each; None means zeros): what Zygote returns through
    mean_and_var over a posterior, for analytic acquisition functions (expected improvement, probability of improvement,
    UCB) and losses on predicted means.  (mean, var) is agp_post_mean_var's on p's handle; the dict comes from one
    agp_post_mean_var_grad call.  Its keys are those of posterior_rand_grad without "Z": the kernel keys, the training
    side "noise", "mean_c" | "mean_v" and "y", the test side "noise_s" (var_bar per point, or its sum for a scalar s2*)
    and "mean_s_v" (mean_bar, CustomMean only); a ConstMean's "mean_c" counts both sides.  inputs=True also returns "x"
    and "xs", shaped like the containers the points came in.  training=False passes NULL for every training-side output
    and returns only the test side ("noise_s", "mean_s_v" and, with inputs=True, "xs"): the call an optimiser over x*
    makes, which does no N x N work.  A CustomMean is treated as a constant of the inputs.  Only a posterior straight
    from posterior(fx0, y) is supported (not a sequentially conditioned one)."""
    p = fx.f
    if not isinstance(p, PosteriorGP) or getattr(p, "fx", None) is None:
        raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "the gradient of mean_and_var over a posterior needs a FiniteGP over "
                       "posterior(fx, y), not over %s" % type(p).__name__)
    eng = engine()
    p, dt, pts, ms, ns, keep = _post_args(fx)
    fx0 = p.fx
    N, M, D = p.data.x.n, pts.n, pts.D

    def cot(a, name):
        if a is None:
            return None
        v = np.ascontiguousarray(np.asarray(a, dtype=dt).ravel())
        if v.shape[0] != M:
            raise DimensionMismatch("%s has %d entries, length(fx) = %d" % (name, v.shape[0], M))
        return v
    mb, vb = cot(mean_bar, "mean_bar"), cot(var_bar, "var_bar")
    mv = _post_call(p, pts, fx.s2)
    f = p.prior
    k = f.kernel
    g, flat = _grad_buffer(k, D, p.data.C.h) if training else (None, None)
    nd = np.empty(N, dtype=dt) if training and np.ndim(fx0.s2) != 0 else None
    md = np.empty(N, dtype=dt) if training and isinstance(f.mean, CustomMean) else None
    yb = np.empty(N, dtype=dt) if training else None
    xg = _points_grad(fx0.x_kind, N, D, dt) if inputs and training else None  # the points go in point-major
    xsg = _points_grad(fx.x_kind, M, D, dt) if inputs else None
    eng.check(eng.L.agp_post_mean_var_grad(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), M, cabi.ptr(mb),
                                           cabi.ptr(vb), None if g is None else g.ctypes.data_as(C.POINTER(C.c_double)),
                                           cabi.ptr(nd), cabi.ptr(md), cabi.ptr(yb), cabi.ptr(xg), cabi.ptr(xsg)))
    res = _grad_result(g, flat, k, D, f.mean, nd, md) if training else {}
    if training:
        res["y"] = yb
    vb64 = np.zeros(M) if vb is None else vb.astype(np.float64)
    res["noise_s"] = vb64 if np.ndim(fx.s2) != 0 else float(np.sum(vb64))
    if isinstance(f.mean, CustomMean):
        res["mean_s_v"] = np.zeros(M) if mb is None else mb.astype(np.float64)
    if inputs:
        if training:
            res["x"] = xg
        res["xs"] = xsg
    return mv, res


def _post_call(p: PosteriorGP, pts: _Points, s2, want_var=True, want_cov=False):
    eng = engine()
    dt = p.data.C.dtype
    pts = pts.astype(dt)
    if pts.D != p.data.x.D:
        raise DimensionMismatch("test points have D=%d, training points D=%d" % (pts.D, p.data.x.D))
    keep = []
    ms = _mean_struct(p.prior.mean.spec(pts, dt), keep)
    mean = np.empty(pts.n, dtype=dt)
    if want_cov:
        cov = np.empty((pts.n, pts.n), dtype=dt, order="F")
        eng.check(eng.L.agp_post_mean_cov(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, C.byref(ms),
                                          cabi.ptr(mean), cabi.ptr(cov)))
        if s2 is not None:
            cov[np.diag_indices(pts.n)] += np.asarray(s2, dtype=dt)
        return mean, cov
    var = np.empty(pts.n, dtype=dt) if want_var else None
    ns = _noise_struct(s2, pts.n, dt, keep) if s2 is not None else None
    eng.check(eng.L.agp_post_mean_var(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, C.byref(ms),
                                      C.byref(ns) if ns is not None else None, cabi.ptr(mean), cabi.ptr(var)))
    return mean, var


def _gram(f: GP, pts: _Points, pts2: Optional[_Points], s2, dt):
    eng = engine()
    keep = []
    pts = pts.astype(dt)
    ks = _kernel_struct(f.kernel, dt, keep, D=pts.D)
    ns = _noise_struct(s2, pts.n, dt, keep) if s2 is not None else None
    if pts2 is None:
        K = np.empty((pts.n, pts.n), dtype=dt, order="F")
        rc = eng.L.agp_gram(eng.h, cabi.dtype_code(dt), C.byref(ks), cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, pts.D,
                            None, 0, C.byref(ns) if ns is not None else None, cabi.ptr(K))
    else:
        pts2 = pts2.astype(dt)
        if pts2.D != pts.D:
            raise DimensionMismatch("inputs have different dimensionality")
        K = np.empty((pts.n, pts2.n), dtype=dt, order="F")
        rc = eng.L.agp_gram(eng.h, cabi.dtype_code(dt), C.byref(ks), cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, pts.D,
                            cabi.ptr(pts2.a), pts2.n, None, cabi.ptr(K))
    eng.check(rc)
    return K


def kernelmatrix(k: Kernel, x, y=None):
    """KernelFunctions.kernelmatrix(k, x[, y]) -- what cov(f, x[, y]) forwards to (src/base_gp.jl:70,74)."""
    pts = _Points(x)
    dt = np.result_type(pts.a.dtype, np.float32)
    return _gram(GP(k), pts, None if y is None else _Points(y), None, dt)


def kernelmatrix_diag(k: Kernel, x):
    """KernelFunctions.kernelmatrix_diag(k, x) -- what var(f, x) forwards to (src/base_gp.jl:72)."""
    return var(GP(k), x)


def mean_vector(m: "MeanFunction", x):
    """mean_vector(m, x) (src/mean_function.jl:27,40,52-55)."""
    pts = _Points(x)
    return m.vector(pts, np.result_type(pts.a.dtype, np.float32))


def _need_x(f, x, name):
    """`mean(f::AbstractGP)` & co. are not defined on purpose (src/abstract_gp.jl:66-87): Julia's ErrorException."""
    if x is None and isinstance(f, AbstractGP):
        raise RuntimeError("`%s(f::AbstractGP)` is not defined (on purpose!).\nPlease provide an `AbstractVector` of locations "
                           "`x` at which you wish to compute your %s vector%s, and call `%s(f(x))`" %
                           (name, name, "s" if name.startswith("mean_and") else "", name))


def mean(f, x=None):
    """mean(fx) (src/finite_gp_projection.jl:53) / mean(f, x) (src/abstract_gp.jl:19)."""
    if isinstance(f, FiniteGP):
        return mean(f.f, f.x)
    _need_x(f, x, "mean")
    pts = _Points(x)
    if isinstance(f, GP):
        return f.mean.vector(pts, np.result_type(pts.a.dtype, np.float32))
    if isinstance(f, PosteriorGP):
        return _post_call(f, pts, None, want_var=False)[0]
    if isinstance(f, ApproxPosteriorGP):
        return _vfe_mean_var(f, pts)[0]
    raise TypeError(type(f))


def cov(f, x=None, z=None):
    """cov(fx) (src/finite_gp_projection.jl:96); cov(f, x[, z]) (src/base_gp.jl:70,74); cov(fx, gx) (:177-180)."""
    if isinstance(f, FiniteGP) and isinstance(x, FiniteGP):
        assert f.f is x.f
        return cov(f.f, f.x, x.x)
    if isinstance(f, FiniteGP):
        if isinstance(f.f, GP):
            return _gram(f.f, f.x, None, f.s2, f.dtype)
        return mean_and_cov(f)[1]
    _need_x(f, x, "cov")
    pts = _Points(x)
    if isinstance(f, GP):
        dt = np.result_type(pts.a.dtype, np.float32)
        return _gram(f, pts, None if z is None else _Points(z), None, dt)
    if isinstance(f, PosteriorGP) and z is None:
        return _post_call(f, pts, None, want_cov=True)[1]
    if isinstance(f, PosteriorGP):  # cov(f_post, x, z) src/exact_gpr_posterior.jl:72-76
        Cx = cov(f.prior, f.data.x, pts)
        Cz = cov(f.prior, f.data.x, _Points(z))
        return cov(f.prior, pts, _Points(z)) - Xt_invA_Y(Cx, f.data.C, Cz)
    if isinstance(f, ApproxPosteriorGP):
        if z is None:  # cov(f_approx_post, x) src/sparse_approximations.jl:187-190
            return _vfe_mean_cov(f, pts)[1]
        # cov(f_approx_post, x, z) (:197-203): the off-diagonal block of the covariance at [x; z]
        zp = _Points(z)
        Cxz = _vfe_mean_cov(f, vcat(pts, zp))[1]
        return np.asfortranarray(Cxz[:pts.n, pts.n:])
    raise TypeError(type(f))


def var(f, x=None):
    """var(fx) (src/finite_gp_projection.jl:114-117) / var(f, x) (src/base_gp.jl:72)."""
    if isinstance(f, FiniteGP):
        return mean_and_var(f)[1]
    _need_x(f, x, "var")
    pts = _Points(x)
    if isinstance(f, GP):
        dt = np.result_type(pts.a.dtype, np.float32)
        k = f.kernel
        if isinstance(k, _CompositeKernel) or k.family > LINEAR:
            return _composite_diag(k if isinstance(k, _CompositeKernel) else KernelSum(k), pts.a.astype(dt))
        if k.family != LINEAR:
            return np.full(pts.n, k.variance, dtype=dt)
        a = pts.a.astype(dt)
        if isinstance(k.transform, ScaleTransform):
            a = a * k.transform.s
        elif isinstance(k.transform, ARDTransform):
            a = a * k.transform.v.astype(dt)
        return (k.variance * ((a * a).sum(1) + k.c)).astype(dt)
    if isinstance(f, PosteriorGP):
        return _post_call(f, pts, None)[1]
    if isinstance(f, ApproxPosteriorGP):
        return _vfe_mean_var(f, pts)[1]
    raise TypeError(type(f))


def mean_and_var(f, x=None):
    """mean_and_var(fx) (src/finite_gp_projection.jl:154-158) -> mean_and_var(f_post, x*)
    (src/exact_gpr_posterior.jl:85-90) + diag(Sigma_y)."""
    if isinstance(f, FiniteGP):
        if isinstance(f.f, PosteriorGP):
            return _post_call(f.f, f.x, f.s2)
        if isinstance(f.f, ApproxPosteriorGP):
            m, v = _vfe_mean_var(f.f, f.x)
            return m, v + f.Sigma_y_diag.astype(v.dtype)
        return mean(f), var(f.f, f.x) + f.Sigma_y_diag
    _need_x(f, x, "mean_and_var")
    return mean(f, x), var(f, x)


def mean_and_cov(f, x=None):
    """mean_and_cov(fx) (src/finite_gp_projection.jl:133-136) / (f_post, x*) (src/exact_gpr_posterior.jl:78-83)."""
    if isinstance(f, FiniteGP):
        if isinstance(f.f, PosteriorGP):
            return _post_call(f.f, f.x, f.Sigma_y_diag, want_cov=True)
        if isinstance(f.f, ApproxPosteriorGP):
            m, Cv = _vfe_mean_cov(f.f, f.x)
            Cv[np.diag_indices(len(f))] += f.Sigma_y_diag.astype(Cv.dtype)
            return m, Cv
        return mean(f), cov(f)
    _need_x(f, x, "mean_and_cov")
    if isinstance(f, PosteriorGP):
        return _post_call(f, _Points(x), None, want_cov=True)
    if isinstance(f, ApproxPosteriorGP):
        return _vfe_mean_cov(f, _Points(x))
    return mean(f, x), cov(f, x)


Normal = namedtuple("Normal", "mu sigma")


def marginals(fx: FiniteGP):
    """marginals(fx) = Normal.(m, sqrt.(c)) (src/finite_gp_projection.jl:203-206) as arrays."""
    m, c = mean_and_var(fx)
    return Normal(m, np.sqrt(c))


def rand(*args):
    """rand([rng,] fx[, S]) (src/finite_gp_projection.jl:233-240): m .+ C.U' * randn(rng, n, S).
    The normals come from the caller's numpy Generator so the stream stays host-defined."""
    args = list(args)
    rng = args.pop(0) if not isinstance(args[0], FiniteGP) else np.random.default_rng()
    fx = args.pop(0)
    S = args.pop(0) if args else None
    if not isinstance(fx.f, (GP, PosteriorGP, ApproxPosteriorGP)):
        raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "sampling from a FiniteGP over %s is outside the device hot path"
                       % type(fx.f).__name__)
    eng = engine()
    dt = fx.f.data.C.dtype if isinstance(fx.f, PosteriorGP) else (fx.f.dtype if isinstance(fx.f, ApproxPosteriorGP) else fx.dtype)
    pts = fx.x.astype(dt)
    ns_cols = 1 if S is None else int(S)
    Z = np.asfortranarray(rng.standard_normal((pts.n, ns_cols)).astype(dt))
    return rand_from_normals(fx, Z, squeeze=S is None)


def rand_from_normals(fx: FiniteGP, Z, squeeze=False):
    if isinstance(fx.f, PosteriorGP):
        return _post_rand_from_normals(fx, Z, squeeze)
    if isinstance(fx.f, ApproxPosteriorGP):
        return _vfe_post_rand_from_normals(fx, Z, squeeze)
    eng = engine()
    f = _prior_of(fx)
    dt = fx.dtype
    pts = fx.x.astype(dt)
    Z = np.asfortranarray(np.asarray(Z, dtype=dt).reshape(pts.n, -1))
    keep = []
    ks = _kernel_struct(f.kernel, dt, keep, D=pts.D)
    ms = _mean_struct(f.mean.spec(pts, dt), keep)
    ns = _noise_struct(fx.s2, pts.n, dt, keep)
    out = np.empty_like(Z, order="F")
    eng.check(eng.L.agp_rand(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), cabi.AGP_POINT_MAJOR,
                             cabi.ptr(pts.a), pts.n, pts.D, cabi.ptr(Z), Z.shape[1], cabi.ptr(out)))
    return out[:, 0] if squeeze else out


def rand_grad(fx: FiniteGP, Z, out_bar, inputs=False):
    """(out, gradient dict) of out = rand_from_normals(fx, Z) = m + C.U' Z over a prior GP, pulled back from the cotangent
    out_bar (the shape of Z: length N or N x S) -- what Zygote returns through the reference's rand(rng, fx, S)
    (test/finite_gp_projection.jl:105-127) for reparameterised Monte Carlo objectives.  The gradient comes from one
    agp_rand_grad call.  The dict has the keys of logpdf_grad ("kernel" for a composite, else "variance", "scale" | "ard",
    "linear_c"; "noise" scalar or per-point; "mean_c" | "mean_v") and "Z", the cotangent of the normals, shaped like Z.
    inputs=True also returns out["x"], the gradient with respect to the input points, shaped like the container fx was
    built from (RowVecs: N x D, ColVecs: D x N, a vector: length N).  A CustomMean is treated as a constant of x: the
    caller chains through out["mean_v"]."""
    if not isinstance(fx.f, GP):
        raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "the gradient of rand is implemented for a FiniteGP over a prior GP, not "
                       "over %s" % type(fx.f).__name__)
    eng = engine()
    f = fx.f
    dt = fx.dtype
    pts = fx.x.astype(dt)
    N, D = pts.n, pts.D
    Zin = np.asarray(Z)
    Zf = np.asfortranarray(np.asarray(Z, dtype=dt).reshape(N, -1))
    Of = np.asfortranarray(np.asarray(out_bar, dtype=dt).reshape(N, -1))
    if Of.shape != Zf.shape:
        raise DimensionMismatch("out_bar has shape %s, Z has %s" % (np.shape(out_bar), Zin.shape))
    S = Zf.shape[1]
    out = rand_from_normals(fx, Zf)
    keep = []
    ks = _kernel_struct(f.kernel, dt, keep, D=D)
    ms = _mean_struct(f.mean.spec(pts, dt), keep)
    ns = _noise_struct(fx.s2, N, dt, keep)
    k = f.kernel
    g, flat = _grad_buffer(k, D)
    nd = np.empty(N, dtype=dt) if np.ndim(fx.s2) != 0 else None
    md = np.empty(N, dtype=dt) if isinstance(f.mean, CustomMean) else None
    zb = np.empty((N, S), dtype=dt, order="F")
    xg = _points_grad(fx.x_kind, N, D, dt) if inputs else None  # the points go in point-major
    eng.check(eng.L.agp_rand_grad(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), cabi.AGP_POINT_MAJOR,
                                  cabi.ptr(pts.a), N, D, cabi.ptr(Zf), S, cabi.ptr(Of),
                                  g.ctypes.data_as(C.POINTER(C.c_double)), cabi.ptr(nd), cabi.ptr(md), cabi.ptr(xg),
                                  cabi.ptr(zb)))
    res = _grad_result(g, flat, k, D, f.mean, nd, md)
    res["Z"] = zb.reshape(Zin.shape) if Zin.ndim == 1 else zb
    if inputs:
        res["x"] = xg
    return (out[:, 0] if Zin.ndim == 1 else out), res


def _posterior_sequential(fx: FiniteGP, y):
    p: PosteriorGP = fx.f
    eng = engine()
    dt = p.data.C.dtype
    pts = fx.x.astype(dt)
    y = np.ascontiguousarray(y, dtype=dt)
    if y.shape[0] != pts.n:
        raise DimensionMismatch("length(fx) != length(y)")
    keep = []
    ms = _mean_struct(p.prior.mean.spec(pts, dt), keep)
    ns = _noise_struct(fx.s2, pts.n, dt, keep)
    n1 = p.data.C.n
    alpha = np.empty(n1 + pts.n, dtype=dt)
    h = C.c_void_p()
    eng.check(eng.L.agp_post_extend(p.data.C.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, cabi.ptr(y), C.byref(ms),
                                    C.byref(ns), cabi.ptr(alpha), C.byref(h)))
    delta = np.concatenate([p.data.delta, y - p.prior.mean.vector(pts, dt)])
    # a NEW device factor: like the reference, the posterior that was conditioned on stays usable
    data = DeviceData(alpha=alpha, C=DeviceCholesky(eng, h, dt), x=vcat(p.data.x, pts), delta=delta)
    return PosteriorGP(p.prior, data)


# ---------------------------------------------------------------------------------------------
# VFE (src/sparse_approximations.jl)
# ---------------------------------------------------------------------------------------------
class VFE:
    """VFE(fz) (src/sparse_approximations.jl:1-12)."""

    def __init__(self, fz: FiniteGP):
        self.fz = fz


class DTC(VFE):
    """DTC(fz) (src/sparse_approximations.jl:14-23): the same optimal approximate posterior as VFE (`posterior(::Union{VFE,DTC}, ...)`
    :58), but `approx_log_evidence` is the DTC objective (:282-286) -- the second output of agp_vfe_elbo."""


def inducing_points(p):
    """inducing_points(f_post_approx) (src/sparse_approximations.jl:219)."""
    return p.approx.fz.x


class ApproxPosteriorGP(AbstractGP):
    """ApproxPosteriorGP(approx, prior, data) (src/sparse_approximations.jl:25-29); `data` lives on the device behind
    the handle, the observations are kept host-side for `update_posterior`."""

    def __init__(self, approx, prior, handle, dtype, x=None, y=None, s2=None):
        self.approx, self.prior, self.h, self.dtype = approx, prior, handle, dtype
        self.x, self.y, self.s2 = x, y, s2

    def __del__(self):
        try:
            if self.h:
                engine().L.agp_vfe_post_free(self.h)
                self.h = None
        except Exception:
            pass


def _vfe_args(vfe: VFE, fx: FiniteGP, y):
    if vfe.fz.f is not fx.f:
        raise AssertionError("vfe.fz.f === fx.f")  # src/sparse_approximations.jl:59,249
    f = _prior_of(fx)
    dt = fx.dtype
    pts, z = fx.x.astype(dt), vfe.fz.x.astype(dt)
    y = np.ascontiguousarray(y, dtype=dt)
    if y.shape[0] != pts.n:
        raise DimensionMismatch("the dimension of the projected GP (here: %d) must equal the number of targets "
                                "(here: %d)" % (pts.n, y.shape[0]))
    keep = [y]
    ks = _kernel_struct(f.kernel, dt, keep, D=pts.D)
    ms = _mean_struct(f.mean.spec(pts, dt), keep)
    ns = _noise_struct(fx.s2, pts.n, dt, keep)
    js = _noise_struct(vfe.fz.s2, z.n, dt, keep)
    return f, dt, pts, z, y, ks, ms, ns, js, keep


def approx_log_evidence(vfe: VFE, fx: FiniteGP, y, return_dtc=False):
    """elbo (src/sparse_approximations.jl:248-254)."""
    eng = engine()
    f, dt, pts, z, y, ks, ms, ns, js, keep = _vfe_args(vfe, fx, y)
    out = np.empty(2, dtype=dt)
    eng.check(eng.L.agp_vfe_elbo(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), cabi.AGP_POINT_MAJOR,
                                 cabi.ptr(pts.a), pts.n, pts.D, cabi.ptr(z.a), z.n, C.byref(js), cabi.ptr(y),
                                 cabi.ptr(out[0:1]), cabi.ptr(out[1:2])))
    if return_dtc:
        return out[0], out[1]
    return out[1] if isinstance(vfe, DTC) else out[0]


def elbo(vfe: VFE, fx: FiniteGP, y):
    """elbo(vfe::VFE, fx, y) = approx_log_evidence(vfe, fx, y) (src/sparse_approximations.jl:254); VFE only."""
    if isinstance(vfe, DTC):
        raise TypeError("elbo is defined for VFE; use approx_log_evidence for DTC")
    return approx_log_evidence(vfe, fx, y)


def approx_log_evidence_grad(vfe: VFE, fx: FiniteGP, y, inputs=False):
    """(value, gradient dict) of approx_log_evidence(vfe, fx, y) -- the elbo for VFE, the DTC objective for DTC -- through
    one agp_vfe_elbo_grad call: what Zygote returns through the reference when a sparse GP is trained.  The dict has the
    keys of logpdf_grad ("variance", "scale" | "ard", "linear_c", "noise" scalar or per-point, "mean_c" | "mean_v") and
    "z", the gradient with respect to the inducing points, shaped like the container vfe.fz was built from (RowVecs: M x D,
    ColVecs: D x M, a vector: length M) in the objective's dtype.  A CustomMean is treated as a constant of x.

    inputs=True also returns out["x"], the gradient with respect to the training inputs, shaped like the container fx was
    built from (RowVecs: N x D, ColVecs: D x N, a vector: length N) in the objective's dtype; everything comes from one
    agp_vfe_elbo_grad_x call.  A CustomMean and per-point noise are treated as constants of x: a caller whose mean or
    noise depends on x chains through out["mean_v"] and out["noise"]."""
    eng = engine()
    f, dt, pts, z, y, ks, ms, ns, js, keep = _vfe_args(vfe, fx, y)
    D = pts.D
    k = f.kernel
    if isinstance(k, _CompositeKernel) or k.family > LINEAR:
        raise AGPError(cabi.AGP_ERR_UNSUPPORTED, "composite kernels are supported on the exact path only (not VFE)")
    value = np.empty(1, dtype=dt)
    g, flat = _grad_buffer(k, D)
    nd = np.empty(pts.n, dtype=dt) if np.ndim(fx.s2) != 0 else None
    md = np.empty(pts.n, dtype=dt) if isinstance(f.mean, CustomMean) else None
    zg = _points_grad(vfe.fz.x_kind, z.n, D, dt)  # the points go in point-major
    objective = 1 if isinstance(vfe, DTC) else 0
    args = (eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n,
            pts.D, cabi.ptr(z.a), z.n, C.byref(js), cabi.ptr(y), objective, cabi.ptr(value),
            g.ctypes.data_as(C.POINTER(C.c_double)), cabi.ptr(nd), cabi.ptr(md), cabi.ptr(zg))
    if inputs:
        xg = _points_grad(fx.x_kind, pts.n, D, dt)
        eng.check(eng.L.agp_vfe_elbo_grad_x(*args, cabi.ptr(xg)))
    else:
        eng.check(eng.L.agp_vfe_elbo_grad(*args))
    out = _grad_result(g, flat, k, D, f.mean, nd, md)
    out["z"] = zg
    if inputs:
        out["x"] = xg
    return value[0], out


def elbo_grad(vfe: VFE, fx: FiniteGP, y, inputs=False):
    """(elbo, gradient dict) of elbo(vfe::VFE, fx, y); VFE only, as elbo.  See approx_log_evidence_grad."""
    if isinstance(vfe, DTC):
        raise TypeError("elbo is defined for VFE; use approx_log_evidence for DTC")
    return approx_log_evidence_grad(vfe, fx, y, inputs=inputs)


def _vfe_posterior(vfe: VFE, fx: FiniteGP, y):
    eng = engine()
    f, dt, pts, z, y, ks, ms, ns, js, keep = _vfe_args(vfe, fx, y)
    h = C.c_void_p()
    eng.check(eng.L.agp_vfe_fit(eng.h, cabi.dtype_code(dt), C.byref(ks), C.byref(ms), C.byref(ns), cabi.AGP_POINT_MAJOR,
                                cabi.ptr(pts.a), pts.n, pts.D, cabi.ptr(z.a), z.n, C.byref(js), cabi.ptr(y), C.byref(h)))
    return ApproxPosteriorGP(vfe, f, h, dt, x=fx.x, y=np.array(y), s2=fx.s2)


def update_posterior(p: ApproxPosteriorGP, a: FiniteGP, y=None):
    """update_posterior(f_post_approx, fx, y) -- new observations, same pseudo-points (src/sparse_approximations.jl:87-119)
    -- and update_posterior(f_post_approx, fz) -- pseudo-points appended (:130-176).  The reference patches its host
    factors with rank-1 / block updates; here the posterior is re-formed by the streamed device fit on the concatenated
    observations / inducing set (one pass over the data, O(N M^2) like the first fit), which yields the same posterior
    (test/sparse_approximations.jl:27-85 compares the two routes to atol 1e-5)."""
    if a.f is not p.prior:
        raise AssertionError("f_post_approx.prior === fx.f")  # :92 / :131
    if y is not None:
        y = np.asarray(y, dtype=p.dtype)
        if y.shape[0] != len(a):
            raise DimensionMismatch("length(fx) != length(y)")
        old_fx = FiniteGP(p.prior, p.x, p.s2)
        s2 = np.concatenate([old_fx.Sigma_y_diag.astype(p.dtype), a.Sigma_y_diag.astype(p.dtype)])
        return _vfe_posterior(p.approx, FiniteGP(p.prior, vcat(p.x, a.x), s2), np.concatenate([p.y, y]))
    fz_old = p.approx.fz
    fz_new = FiniteGP(p.prior, vcat(fz_old.x, a.x), fz_old.s2 if np.ndim(fz_old.s2) == 0 else
                      np.concatenate([np.asarray(fz_old.s2), a.Sigma_y_diag]))
    return _vfe_posterior(type(p.approx)(fz_new), FiniteGP(p.prior, p.x, p.s2), p.y)


def _vfe_mean_var(p: ApproxPosteriorGP, pts: _Points):
    eng = engine()
    pts = pts.astype(p.dtype)
    m = np.empty(pts.n, dtype=p.dtype)
    v = np.empty(pts.n, dtype=p.dtype)
    eng.check(eng.L.agp_vfe_mean_var(p.h, cabi.AGP_POINT_MAJOR, cabi.ptr(pts.a), pts.n, cabi.ptr(m), cabi.ptr(v)))
    if isinstance(p.prior.mean, CustomMean):  # the handle carries Zero/Const means only: a closure is evaluated here
        m = m + p.prior.mean.vector(pts, p.dtype)
    return m, v
