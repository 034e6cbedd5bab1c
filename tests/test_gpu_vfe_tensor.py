"""The VFE path (`agp_vfe_elbo` / `agp_vfe_fit` and the predictions of its handle) at the sizes where it runs on the tensor
cores, against the fp64 oracle (oracle/agp_ref.py, pinned at M = 1100 by tests/test_oracle_vfe_scale.py):

* D += A_c A_c' as ONE long-K int8-slice product per chunk (m_pad >= 1024 and a chunk of 1024 columns or more),
* A_c = L_z^-1 K_zx and the prediction solves on the tensor forward substitution (m_pad >= 2048, 512 columns or more),
* a stream of several chunks: int8 chunks and a tile-GEMM tail accumulated into the same D, a one-column last chunk,
  the per-chunk offsets of the noise and residual vectors, the slice workspace re-created for a last chunk of another K,
* K_zz and D + I factored on the int8-slice Cholesky (fp32, m_pad >= 4096).

Which path ran is asserted from the launch counter: an int8 product is three launches (row scales, slices, update) where
the tile GEMM is one, and the two-level substitution has its own launch pattern (`_subst_launches`).  The counter is
compared between the automatic policy and tensor mode 0 on the same problem, so a threshold that moves a case off its
branch fails the case.  (The `elbo` bits themselves are no evidence: its scalars leave their CTAs through fp64 atomics
and vary in the last bits between two identical calls.)

Tolerances: elbo / dtc rtol 1e-8 (fp64) and 1e-4 (fp32), what BASELINE.json and bench.py demand."""
import numpy as np
import pytest

from oracle import agp_ref as ref

pytestmark = pytest.mark.gpu

TILE = 128
EPS32 = float(np.finfo(np.float32).eps)


def _rup(x, m=TILE):
    return (x + m - 1) // m * m


@pytest.fixture
def eng(ag):
    """the engine under the automatic policy; whatever a case sets is put back"""
    e = ag.engine()
    c = e.get_config()
    old = (c.fp64_mode, c.fp32_mode, c.tile_nb)
    assert old == (-1, -1, 0), "automatic policy expected"
    yield e
    e.set_config(fp64_mode=old[0], fp32_mode=old[1], tile_nb=old[2])


class Problem:
    """C5-like data (16 features, SqExponential, lengthscale 2, inducing points drawn from the data) with M chosen by the
    case; `variant` swaps the kernel, the mean and the noise.  The oracle always sees the fp64 image of the same bytes."""

    def __init__(self, ag, n, m, dtype, variant="c5", seed=7):
        cfg = ref.make_config("C5", n=n, dtype=dtype)
        self.ag, self.dtype, self.n, self.m = ag, dtype, n, m
        self.X, self.y = cfg["X"], cfg["y"]
        self.Z = self.X[np.random.default_rng(seed).permutation(n)[:m]].copy()
        self.jit = 1e-6 if dtype == np.float64 else 1e-4
        d = self.X.shape[1]
        self.k, self.kern = cfg["k"], ag.SqExponentialKernel().compose(ag.ScaleTransform(cfg["k"].scale))
        self.mean_ref, self.mean_ag = ref.MeanSpec(), None
        self.noise_ref, self.s2 = ref.NoiseSpec(0, 0.1), 0.1
        rng = np.random.default_rng(seed + 1)
        if variant in ("noise_vector_const_mean", "matern32_noise_vector"):
            self.s2 = (0.05 + 0.1 * rng.random(n)).astype(dtype)
            self.noise_ref = ref.NoiseSpec(1, v=self.s2.astype(np.float64))
        if variant == "noise_vector_const_mean":
            self.mean_ref, self.mean_ag = ref.MeanSpec(1, 0.3), 0.3
        if variant == "matern32_noise_vector":
            self.k = ref.KernelSpec(ref.MATERN32, 1.3, ref.T_SCALE, scale=0.6)
            self.kern = 1.3 * ag.Matern32Kernel().compose(ag.ScaleTransform(0.6))
        if variant == "ard_vector_mean":
            w = ((0.5 * (1.0 + 0.5 * np.arange(d) / d))).astype(dtype)
            self.k = ref.KernelSpec(ref.SE, 1.0, ref.T_ARD, ard=w.astype(np.float64))
            self.kern = ag.SqExponentialKernel().compose(ag.ARDTransform(w))
            def mean_fn(xi):  # per-point mean: shipped as a vector, offset per chunk like the noise
                return 0.2 * np.cos(3.0 * float(xi[0]))
            mv = np.array([mean_fn(xi) for xi in self.X], dtype=dtype)
            self.mean_ref = ref.MeanSpec(2, v=mv.astype(np.float64))
            self.mean_ag = ag.CustomMean(mean_fn)

    def permuted(self, perm):
        import copy
        q = copy.copy(self)
        q.X, q.y = self.X[perm].copy(), self.y[perm].copy()
        if np.ndim(self.s2):
            q.s2 = self.s2[perm].copy()
            q.noise_ref = ref.NoiseSpec(1, v=q.s2.astype(np.float64))
        return q

    def _f(self):
        ag = self.ag
        return ag.GP(self.kern) if self.mean_ag is None else ag.GP(self.mean_ag, self.kern)

    def _vfe_fx(self, f, jit=None):
        ag = self.ag
        return ag.VFE(f(ag.RowVecs(self.Z), self.jit if jit is None else jit)), f(ag.RowVecs(self.X), self.s2)

    def elbo(self):
        """(elbo, dtc) of the device and the number of kernel launches the call made"""
        f = self._f()
        vfe, fx = self._vfe_fx(f)
        e = self.ag.engine()
        l0 = e.launch_count()
        el, dt = self.ag.approx_log_evidence(vfe, fx, self.y, return_dtc=True)
        assert el.dtype == self.dtype
        return float(el), float(dt), e.launch_count() - l0

    def posterior(self):
        vfe, fx = self._vfe_fx(self._f())
        return self.ag.posterior(vfe, fx, self.y)

    def _ref_args(self):
        return (self.k, self.mean_ref, self.noise_ref, self.X.astype(np.float64), self.y.astype(np.float64),
                self.Z.astype(np.float64), ref.NoiseSpec(0, self.jit))

    def oracle(self):
        """(elbo, dtc) in fp64, src/sparse_approximations.jl:248-254 and :282-286 from ONE pass over the intermediates"""
        a = self._ref_args()
        dt, A = ref._compute_intermediates(*a)
        return float(dt - (ref.tr_Cf_invSy(a[0], a[2], a[3]) - np.sum(A * A)) / 2.0), float(dt)

    def oracle_posterior(self):
        return ref.vfe_posterior(*self._ref_args())

    def cond_kzz(self):
        Kzz = ref.kernelmatrix(self.k, self.Z.astype(np.float64))
        Kzz[np.diag_indices(self.m)] += self.jit
        return float(np.linalg.cond(Kzz))


def _rtol(dtype):
    return 1e-8 if dtype == np.float64 else 1e-4


def _close(got, want, rtol):
    return abs(got - want) <= rtol * abs(want)


def _chunks(n, m_pad, dtype, chunk=None, tensor=True):
    """the chunk widths `vfe_core` streams (padded to 128); the long-K product (m_pad >= 1024) caps them at 32 768"""
    tc = tensor and m_pad >= 1024
    cap = chunk if chunk else int(2.0e9 / (m_pad * np.dtype(dtype).itemsize))
    cap = max(TILE, cap // TILE * TILE)
    cap = min(cap, _rup(n) + TILE)
    if tc:
        cap = min(cap, 32768)
    return [_rup(min(cap, n - c0)) for c0 in range(0, n, cap)]


def _subst_launches(m_pad, ncols, tensor):
    """launches of one multi-column forward substitution V <- L^-1 V: 128-steps (solve + update below) on the tile GEMM, or
    512-row outer blocks whose rank-512 update of everything below is an int8 product (2 + 2 + 1 launches)"""
    nblk = m_pad // TILE
    if not (tensor and m_pad >= 2048 and ncols % TILE == 0 and ncols >= 512):
        return 2 * nblk - 1
    total = 0
    for ko in range(0, nblk, 4):
        nb = min(4, nblk - ko)
        total += 2 * nb - 1
        if ko + nb < nblk:
            total += 5 if nb == 4 else 1
    return total


def _stream_delta(n, m_pad, dtype, chunk=None):
    """launches the tensor paths ADD to the data stream of one elbo call over tensor mode 0, and the number of int8 chunks"""
    def launches(tensor):  # per chunk: Gram, column scaling, substitution, product (3 or 1), gemv, sum of squares
        ws = _chunks(n, m_pad, dtype, chunk, tensor)
        return sum(4 + _subst_launches(m_pad, w, tensor) + (3 if tensor and m_pad >= 1024 and w >= 1024 else 1) for w in ws)
    widths = _chunks(n, m_pad, dtype, chunk)
    int8 = [w for w in widths if m_pad >= 1024 and w >= 1024]
    return launches(True) - launches(False), len(int8), len(widths)


def _elbo_on_and_off(eng, p):
    """the same call under the automatic policy and with the tensor paths off"""
    on = p.elbo()
    eng.set_config(fp64_mode=0, fp32_mode=0)
    off = p.elbo()
    eng.set_config(fp64_mode=-1, fp32_mode=-1)
    return on, off


# ---- one chunk ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("m", [1100, 1024, 1025])
def test_long_k_syrk_alone(ag, eng, dtype, m):
    """m_pad in [1024, 2047], one chunk of 3072 columns: only D += A A' differs between the modes (the substitution and both
    factorisations stay on the tile kernels), so this isolates the long-K product and its operands: leading dimensions,
    lower-only tiles into the fp32 / fp64 D, the identity-padded rows (M = 1025: 127 of them) and the 72 zero columns."""
    p = Problem(ag, 3000, m, dtype)
    (el, dt, l_on), (el0, dt0, l_off) = _elbo_on_and_off(eng, p)
    delta, n_int8, n_chunks = _stream_delta(3000, _rup(m), dtype)
    assert (n_int8, n_chunks, delta) == (1, 1, 2)
    assert l_on - l_off == 2, (l_on, l_off)
    el_r, dt_r = p.oracle()
    print("syrk alone", dtype.__name__, m, (el - el_r) / abs(el_r), (dt - dt_r) / abs(dt_r), (el0 - el_r) / abs(el_r))
    assert _close(el, el_r, _rtol(dtype)) and _close(dt, dt_r, _rtol(dtype)), (el, el_r, dt, dt_r)
    assert _close(el0, el_r, _rtol(dtype)) and _close(dt0, dt_r, _rtol(dtype)), (el0, el_r, dt0, dt_r)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("m", [2304, 2100])
def test_syrk_and_tensor_substitution(ag, eng, dtype, m):
    """m_pad >= 2048: A = L_z^-1 K_zx on the two-level substitution too; the predictions of the handle solve against U and
    Lambda the same way (1536 points for mean_and_var, 600 for the full covariance and the FiniteGP over it)."""
    n, m_pad = 6000, _rup(m)
    p = Problem(ag, n, m, dtype)
    (el, dt, l_on), (el0, dt0, l_off) = _elbo_on_and_off(eng, p)
    delta, n_int8, n_chunks = _stream_delta(n, m_pad, dtype)
    assert (n_int8, n_chunks) == (1, 1) and delta > 2
    assert l_on - l_off == delta, (l_on, l_off, delta)
    el_r, dt_r = p.oracle()
    print("syrk+subst", dtype.__name__, m, (el - el_r) / abs(el_r), (dt - dt_r) / abs(dt_r), (el0 - el_r) / abs(el_r))
    assert _close(el, el_r, _rtol(dtype)) and _close(dt, dt_r, _rtol(dtype)), (el, el_r, dt, dt_r)

    vp, vr = p.posterior(), p.oracle_posterior()
    rng = np.random.default_rng(3)
    Xs = rng.random((1536, p.X.shape[1])).astype(dtype)
    Xs64 = Xs.astype(np.float64)
    l0 = eng.launch_count()
    mu, v = ag.mean_and_var(vp, ag.RowVecs(Xs))
    l_on = eng.launch_count() - l0
    eng.set_config(fp64_mode=0, fp32_mode=0)
    l0 = eng.launch_count()
    mu0, v0 = ag.mean_and_var(vp, ag.RowVecs(Xs))
    l_off = eng.launch_count() - l0
    eng.set_config(fp64_mode=-1, fp32_mode=-1)
    # mean_and_var(f, x) is mean(f, x) and var(f, x): two calls, each two substitutions (U, then Lambda) of 1536 columns
    assert l_on - l_off == 4 * (_subst_launches(m_pad, 1536, True) - _subst_launches(m_pad, 1536, False)), (l_on, l_off)
    assert not np.array_equal(mu, mu0)  # no atomics on this path: different bits mean a different kernel ran
    mu_r, v_r = ref.vfe_mean_and_var(vr, Xs64)
    if dtype == np.float64:
        tol_m = tol_v = dict(rtol=1e-6, atol=1e-7)
    else:
        # fp32 bound from the case.  Every prediction is a function of a = L^-1 k(z, x*), L L' = K_zz + J.  The substitution
        # is backward stable: the computed a solves (L + dL) a = k with |dL| <= g |L|, so |da| / |a| <= g cond(L) =
        # g sqrt(cond(K_zz + J)).  Everything after it contracts: Lambda Lambda' = A A' + I >= I, so |Lambda^-1 a| <= |a|,
        # and |a|^2 <= k(x*, x*) = 1.  The same error sits in the columns of A the fit streamed.  The worst case is
        # g = M eps32; rounding errors of both signs leave far less, and g = 4 eps32 is the bound held here: on the H100
        # the means are off by 0.45 eps32 sqrt(cond) and the variances by 0.003 eps32 sqrt(cond) (cond = 1.5e7, M = 2304).
        # A mean is a' m_e, so its bound carries the size of the oracle's means; a variance is bounded by k** = 1.
        bound = 4 * EPS32 * np.sqrt(p.cond_kzz())
        tol_m = dict(rtol=0, atol=bound * max(1.0, float(np.abs(mu_r).max())))
        tol_v = dict(rtol=0, atol=bound)
        print("fp32 prediction bound", m, bound, float(np.abs(mu - mu_r).max()), float(np.abs(v - v_r).max()))
    assert np.allclose(mu, mu_r, **tol_m), float(np.abs(mu - mu_r).max())
    assert np.allclose(v, v_r, **tol_v), float(np.abs(v - v_r).max())
    assert np.allclose(mu0, mu_r, **tol_m) and np.allclose(v0, v_r, **tol_v)

    # full covariance, and logpdf / rand of a FiniteGP over the approximate posterior (600 points: 640 padded columns)
    Xc, Xc64 = Xs[:600], Xs64[:600]
    l0 = eng.launch_count()
    mc, Cc = ag.mean_and_cov(vp, ag.RowVecs(Xc))
    l_on = eng.launch_count() - l0
    eng.set_config(fp64_mode=0, fp32_mode=0)
    l0 = eng.launch_count()
    mc0, Cc0 = ag.mean_and_cov(vp, ag.RowVecs(Xc))
    l_off = eng.launch_count() - l0
    eng.set_config(fp64_mode=-1, fp32_mode=-1)
    assert l_on - l_off == 2 * (_subst_launches(m_pad, 640, True) - _subst_launches(m_pad, 640, False)), (l_on, l_off)
    mr, Cr = ref.vfe_mean_and_cov(vr, Xc64)
    assert np.allclose(mc, mr, **tol_m), float(np.abs(mc - mr).max())
    assert np.allclose(Cc, Cr, **tol_v), float(np.abs(Cc - Cr).max())
    assert np.allclose(Cc0, Cr, **tol_v)
    s2 = 0.05
    U = ref.cholesky_upper(Cr + s2 * np.eye(600))
    Ys = (mr[:, None] + U.T @ rng.standard_normal((600, 2))).astype(dtype)
    want = -0.5 * (600 * ref.LOG2PI + ref.logdet_chol(U) + ref.diag_Xt_invA_X(U, Ys.astype(np.float64) - mr[:, None]))
    got = ag.logpdf(vp(ag.RowVecs(Xc), s2), Ys)
    print("vfe post logpdf", dtype.__name__, m, got, want)
    # the value is a small difference of terms of size 600 log(2 pi) / 2: fp32 is held to 1e-4 of the terms, not of the rest
    lp_tol = 1e-8 * np.abs(want) if dtype == np.float64 else 1e-4 * (300 * ref.LOG2PI + np.abs(want))
    assert np.all(np.abs(got - want) <= lp_tol), (got, want)
    Zn = rng.standard_normal((600, 3)).astype(dtype)
    got_r = ag.rand_from_normals(vp(ag.RowVecs(Xc), s2), Zn)
    want_r = mr[:, None] + U.T @ Zn.astype(np.float64)
    atol_r = 1e-7 if dtype == np.float64 else tol_m["atol"] + 4 * tol_v["atol"] / np.sqrt(s2)
    assert np.allclose(got_r, want_r, rtol=0, atol=atol_r), float(np.abs(got_r - want_r).max())


# ---- several chunks ---------------------------------------------------------------------------------------------------
STREAMS = [(2500, 1024), (2305, 1152), (2500, 128), (2560, 1024), (2500, 1536)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_stream_edges_forced_chunks(ag, eng, dtype, monkeypatch):
    """AGP_VFE_CHUNK forces the chunk width at M = 1100: 1024 + 1024 + a 452-column tail on the tile GEMM mixed into one D;
    1152 + 1152 + ONE column; 128-column chunks (all on the GEMM); N a multiple of 128; 1536 + 1024 (the slice workspace
    re-created for the other K).  Each matches the oracle, and every chunking of the same N agrees with the one-chunk
    result: the order of the sums changes, nothing else."""
    m, m_pad = 1100, 1152
    want_int8 = {(2500, 1024): (2, 3), (2305, 1152): (2, 3), (2500, 128): (0, 20), (2560, 1024): (2, 3), (2500, 1536): (2, 2)}
    one, oracle, one_off_launches = {}, {}, {}
    for n, chunk in STREAMS:
        p = Problem(ag, n, m, dtype)
        if n not in one:
            one[n], off_one = _elbo_on_and_off(eng, p)
            oracle[n], one_off_launches[n] = p.oracle(), off_one[2]
            assert _stream_delta(n, m_pad, dtype)[1:] == (1, 1)
        monkeypatch.setenv("AGP_VFE_CHUNK", str(chunk))
        (el, dt, l_on), (el0, dt0, l_off) = _elbo_on_and_off(eng, p)
        monkeypatch.delenv("AGP_VFE_CHUNK")
        delta, n_int8, n_chunks = _stream_delta(n, m_pad, dtype, chunk)
        assert (n_int8, n_chunks) == want_int8[(n, chunk)] and delta == 2 * n_int8
        assert l_on - l_off == delta, (n, chunk, l_on, l_off)
        # a chunk on the tile kernels is Gram, column scaling, 2 * 9 - 1 substitution steps, GEMM, gemv and sum of squares
        assert l_off - one_off_launches[n] == (n_chunks - 1) * (2 * (m_pad // TILE) + 4), (n, chunk, l_off, one_off_launches[n])
        el_r, dt_r = oracle[n]
        agree = 1e-10 if dtype == np.float64 else 1e-5
        print("stream", dtype.__name__, n, chunk, (el - el_r) / abs(el_r), (el - one[n][0]) / abs(el_r), (dt - one[n][1]) / abs(dt_r))
        assert _close(el, el_r, _rtol(dtype)) and _close(dt, dt_r, _rtol(dtype)), (n, chunk, el, el_r, dt, dt_r)
        assert _close(el, one[n][0], agree) and _close(dt, one[n][1], agree), (n, chunk, el, one[n][0], dt, one[n][1])
        assert _close(el0, one[n][0], agree) and _close(dt0, one[n][1], agree), (n, chunk, el0, one[n][0])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_real_chunk_boundary(ag, eng, dtype):
    """no knob: N = 40 000 at M = 1100 streams 32 768 + 7232 columns, so the int8 product runs at its largest K (the bound
    of its int32 accumulators) and the slice workspace is re-created for K = 7296."""
    n, m = 40000, 1100
    p = Problem(ag, n, m, dtype)
    assert _chunks(n, 1152, dtype) == [32768, 7296] and _chunks(n, 1152, dtype, tensor=False) == [40064]
    (el, dt, l_on), (el0, dt0, l_off) = _elbo_on_and_off(eng, p)
    # two int8 products, and one chunk more than the tile kernels need (they take all 40 000 columns at once)
    assert _stream_delta(n, 1152, dtype)[0] == 4 + 22
    assert l_on - l_off == 26, (l_on, l_off)
    el_r, dt_r = p.oracle()
    print("boundary", dtype.__name__, (el - el_r) / abs(el_r), (dt - dt_r) / abs(dt_r), (el0 - el_r) / abs(el_r))
    assert _close(el, el_r, _rtol(dtype)) and _close(dt, dt_r, _rtol(dtype)), (el, el_r, dt, dt_r)
    assert _close(el0, el_r, _rtol(dtype)) and _close(dt0, dt_r, _rtol(dtype)), (el0, el_r, dt0, dt_r)


def test_c5_shape_scaled_fp32(ag, eng):
    """what bench.py's parity key samples: fp32, N = 20 000, M = 4224 -- K_zz and D + I factored by the int8-slice Cholesky
    (m_pad >= 4096, 512-wide panels), the substitution and the long-K product on the tensor cores."""
    n, m = 20000, 4224
    p = Problem(ag, n, m, np.float32)
    (el, dt, l_on), (el0, dt0, l_off) = _elbo_on_and_off(eng, p)
    delta, n_int8, n_chunks = _stream_delta(n, m, np.float32)
    assert (n_int8, n_chunks) == (1, 1)
    # the stream accounts for `delta`.  The rest is the two factorisations: at 33 blocks the int8-slice Cholesky (512-wide
    # outer panels, one sliced trailing update each) makes 40 launches FEWER than the 128-wide tile schedule -- a count
    # measured on the H100, not derived; it moves if either factorisation leaves the int8 path
    assert l_on - l_off == delta - 2 * 40, (l_on, l_off, delta)
    el_r, dt_r = p.oracle()
    print("c5 scaled", (el - el_r) / abs(el_r), (dt - dt_r) / abs(dt_r), (el0 - el_r) / abs(el_r), el_r, dt_r)
    assert _close(el, el_r, 1e-4) and _close(dt, dt_r, 1e-4), (el, el_r, dt, dt_r)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("variant", ["noise_vector_const_mean", "ard_vector_mean", "matern32_noise_vector"])
def test_variants_over_two_chunks(ag, eng, dtype, variant, monkeypatch):
    """per-point noise, constant and per-point mean, ARD weights, Matern-3/2 at M = 1100 over chunks of 1536 + 964 columns:
    the noise scales and the residuals are offset per chunk, and only a per-point vector can tell a wrong offset."""
    n, m = 2500, 1100
    p = Problem(ag, n, m, dtype, variant)
    monkeypatch.setenv("AGP_VFE_CHUNK", "1536")
    (el, dt, l_on), (el0, dt0, l_off) = _elbo_on_and_off(eng, p)
    monkeypatch.delenv("AGP_VFE_CHUNK")
    assert l_on - l_off == 4, (l_on, l_off)
    el_r, dt_r = p.oracle()
    print("variant", dtype.__name__, variant, (el - el_r) / abs(el_r), (dt - dt_r) / abs(dt_r))
    assert _close(el, el_r, _rtol(dtype)) and _close(dt, dt_r, _rtol(dtype)), (el, el_r, dt, dt_r)


def test_permuting_the_data_leaves_elbo_unchanged(ag, eng, monkeypatch):
    """X, y and the noise vector permuted together, three chunks (two int8, one GEMM): a point lost in a padding column or a
    chunk counted twice breaks this whatever the oracle says."""
    n, m = 2500, 1100
    p = Problem(ag, n, m, np.float64, "noise_vector_const_mean")
    q = p.permuted(np.random.default_rng(11).permutation(n))
    monkeypatch.setenv("AGP_VFE_CHUNK", "1024")
    el, dt, l1 = p.elbo()
    el2, dt2, l2 = q.elbo()
    eng.set_config(fp64_mode=0)
    l_off = p.elbo()[2]
    eng.set_config(fp64_mode=-1)
    monkeypatch.delenv("AGP_VFE_CHUNK")
    assert l1 == l2 and l1 - l_off == 4
    print("permutation", (el - el2) / abs(el), (dt - dt2) / abs(dt))
    assert _close(el2, el, 1e-10) and _close(dt2, dt, 1e-10), (el, el2, dt, dt2)


def test_not_posdef_on_the_large_path_then_reuse(ag, eng):
    """64 duplicated inducing points and no jitter at M = 1100: PosDefException (an error return, the half-built handle is
    freed), and the next call on the same engine, through the same slice workspace, is right."""
    p = Problem(ag, 3000, 1100, np.float64)
    good = p.elbo()
    Z = p.Z.copy()
    p.Z = Z.copy()
    p.Z[-64:] = Z[:64]
    f = p._f()
    for call in (lambda v, fx: ag.approx_log_evidence(v, fx, p.y), lambda v, fx: ag.posterior(v, fx, p.y)):
        with pytest.raises(ag.PosDefException):
            call(*p._vfe_fx(f, jit=0.0))
    p.Z = Z
    again = p.elbo()
    assert again[2] == good[2]
    assert _close(again[0], good[0], 1e-12) and _close(again[1], good[1], 1e-12), (good, again)
    el_r, dt_r = p.oracle()
    assert _close(again[0], el_r, 1e-8) and _close(again[1], dt_r, 1e-8)


def test_workspaces_survive_other_sizes(ag, eng):
    """one engine: elbo at (M = 1100, N = 3000), then (M = 2304, N = 6000) -- both slice workspaces resized -- then an exact
    fit with 1536-point predictions (resizes the factorisation's workspace again), then the first elbo again.  A stale slice
    buffer or row scale left by a resize shows here.  The elbo scalars are summed with fp64 atomics, so the two results
    agree to 1e-12, not bit for bit; the predictions of a handle kept from the start have no atomics and must not move."""
    p = Problem(ag, 3000, 1100, np.float64)
    first = p.elbo()
    vp = p.posterior()
    Xs = np.random.default_rng(5).random((1536, 16))
    mu, v = ag.mean_and_var(vp, ag.RowVecs(Xs))
    big = Problem(ag, 6000, 2304, np.float64)
    big_first = big.elbo()
    f = ag.GP(p.kern)
    post = ag.posterior(f(ag.RowVecs(p.X), 0.1), p.y)
    ag.mean_and_var(post, ag.RowVecs(Xs))
    last = p.elbo()
    assert last[2] == first[2]
    assert _close(last[0], first[0], 1e-12) and _close(last[1], first[1], 1e-12), (first, last)
    mu2, v2 = ag.mean_and_var(vp, ag.RowVecs(Xs))
    assert np.array_equal(mu, mu2) and np.array_equal(v, v2)
    big_last = big.elbo()
    assert _close(big_last[0], big_first[0], 1e-12) and _close(big_last[1], big_first[1], 1e-12), (big_first, big_last)
    el_r, dt_r = p.oracle()
    assert _close(last[0], el_r, 1e-8) and _close(last[1], dt_r, 1e-8)
