"""The int8-sliced tensor-core (wgmma) factorisation checked IN PLACE: `agp_fit` driven through the path that runs every
n_pad >= 8192 fit (fp64_mode = 1, 512-wide outer panels, slicing, persistent trailing update, look-ahead) against the
oracle -- logpdf rtol 1e-8 as BASELINE.json demands, alpha and the factor U -- plus the block-cyclic strip-table tile
enumeration of the multi-GPU trailing update, driven on ONE device through `agp_debug_ozaki_syrk_map` exactly as
`fit_dist_impl` calls it, against a torch fp64 matmul.
Reference operations: cholesky at /root/reference/src/finite_gp_projection.jl:308 and
/root/reference/src/exact_gpr_posterior.jl:31; logpdf :306-311; posterior src/exact_gpr_posterior.jl:29-35."""
import ctypes as C

import numpy as np
import pytest

from oracle import agp_ref as ref

pytestmark = pytest.mark.gpu


def _fit(ag, cfg):
    f = ag.GP(ag.SqExponentialKernel().compose(ag.ScaleTransform(cfg["k"].scale)))
    return ag.fit(f(ag.RowVecs(cfg["X"]), cfg["noise"].s), cfg["y"])


@pytest.fixture
def forced_tcgen05(ag):
    eng = ag.engine()
    c0 = eng.get_config()
    old = (c0.fp64_mode, c0.tile_nb)
    eng.set_config(fp64_mode=1, tile_nb=512)
    yield eng
    eng.set_config(fp64_mode=old[0], tile_nb=old[1])


@pytest.mark.parametrize("n", [1300, 2304, 4096])
def test_fit_forced_tcgen05_matches_oracle(ag, forced_tcgen05, n):
    """below the automatic threshold the engine is forced onto the int8-slice path (the C2 workload at n = 4096)"""
    eng = forced_tcgen05
    cfg = ref.make_config("C2", n=n)
    lp, post = _fit(ag, cfg)
    lp_ref = ref.logpdf(cfg["k"], cfg["mean"], cfg["noise"], cfg["X"], cfg["y"])
    pr = ref.posterior(cfg["k"], cfg["mean"], cfg["noise"], cfg["X"], cfg["y"])
    assert abs(lp - lp_ref) <= 1e-8 * abs(lp_ref), (lp, lp_ref)
    a = post.data.alpha
    assert np.allclose(a, pr["alpha"], rtol=1e-6, atol=1e-7 * np.abs(pr["alpha"]).max())
    assert np.isclose(post.data.C.logdet(), ref.logdet_chol(pr["U"]), rtol=1e-9)
    if n <= 2304:
        assert np.allclose(post.data.C.U, pr["U"], rtol=1e-7, atol=1e-9)
    # the int8-slice path really ran: its 2^-49 slice truncation makes it differ from the DMMA path in the last bits
    eng.set_config(fp64_mode=0, tile_nb=0)
    lp0, post0 = _fit(ag, cfg)
    eng.set_config(fp64_mode=1, tile_nb=512)
    assert not np.array_equal(a, post0.data.alpha)
    assert abs(lp - lp0) <= 1e-9 * abs(lp0)


@pytest.mark.parametrize("n,d", [(8192, 16), (8320, 8), (16384, 8)])
def test_fit_auto_mode_large_matches_oracle(ag, n, d):
    """automatic policy (n_pad >= 8192 -> int8 slices, 512-wide panels): the path of every C4 number.  n = 8320 has a ragged
    last outer panel (n_pad % 512 = 128): int8-slice panels followed by a DMMA tail."""
    cfg = ref.make_config("C4", n=n)
    cfg["X"] = np.ascontiguousarray(cfg["X"][:, :d])
    cfg["k"] = ref.KernelSpec(ref.SE, 1.0, ref.T_SCALE, scale=1.0 / (0.5 * np.sqrt(d)))
    c = ag.engine().get_config()
    assert c.fp64_mode < 0 and c.tile_nb == 0, "default (auto) policy expected"
    lp, post = _fit(ag, cfg)
    lp_ref = ref.logpdf(cfg["k"], cfg["mean"], cfg["noise"], cfg["X"], cfg["y"])
    assert abs(lp - lp_ref) <= 1e-8 * abs(lp_ref), (lp, lp_ref)
    pr = ref.posterior(cfg["k"], cfg["mean"], cfg["noise"], cfg["X"], cfg["y"])
    assert np.allclose(post.data.alpha, pr["alpha"], rtol=1e-6, atol=1e-7 * np.abs(pr["alpha"]).max())
    assert np.isclose(post.data.C.logdet(), ref.logdet_chol(pr["U"]), rtol=1e-9)
    Xs = np.random.default_rng(9).random((300, d))
    m, v = ag.mean_and_var(post, ag.RowVecs(Xs))
    m_r, v_r = ref.post_mean_and_var(pr, Xs)
    assert np.allclose(m, m_r, rtol=1e-6, atol=1e-7) and np.allclose(v, v_r, rtol=1e-6, atol=1e-8)


@pytest.mark.parametrize("R,me,kk,nto,W", [(2, 0, 0, 9, 512), (2, 1, 2, 9, 512), (4, 3, 1, 11, 512), (8, 5, 0, 17, 256),
                                          (8, 0, 3, 20, 512), (4, 2, 0, 6, 128)])
def test_strip_table_enumeration_matches_fp64(ag, R, me, kk, nto, W):
    """trailing update of outer step kk on rank `me` of a 1 x R block-column-cyclic grid (fit_dist_impl's `trailing`):
    local columns = the outer blocks j > kk with j % R == me, packed; rows = everything below panel kk (+128 border)."""
    import torch
    eng = ag.engine()
    K, S = W, 7
    rows_below = (nto - (kk + 1)) * W + 128
    loc = [j for j in range(kk + 1, nto) if j % R == me]
    if not loc:
        pytest.skip("rank owns no trailing block")
    ncols = len(loc) * W
    g = torch.Generator(device="cuda").manual_seed(R * 100 + me * 10 + kk)
    P = (torch.rand((K, rows_below), generator=g, device="cuda", dtype=torch.float64) * 2 - 1)
    P = P * torch.logspace(-2, 2, rows_below, device="cuda", dtype=torch.float64)[None, :]   # storage of col-major rows_below x K
    ldc = rows_below + 3
    Cst = torch.rand((ncols, ldc), generator=g, device="cuda", dtype=torch.float64)           # storage of col-major ldc x ncols
    C0 = Cst.clone()
    b_off = (loc[0] - (kk + 1)) * W
    torch.cuda.synchronize()  # the library works on its own stream: device inputs must be complete before the call
    rc = eng.L.agp_debug_ozaki_syrk_map(eng.h, C.c_void_p(Cst.data_ptr()), ldc, C.c_void_p(P.data_ptr()), rows_below,
                                        rows_below, rows_below, ncols, K, S, R * W, W, b_off, 0)
    eng.check(rc)
    Pm = P.t()                                                  # rows_below x K
    n = torch.arange(ncols, device="cuda")
    src = (n // W) * (R * W) + n % W + b_off                    # panel row paired with local column n
    want = C0.t()[:rows_below] - Pm @ Pm[src].t()               # rows_below x ncols
    got = Cst.t()[:rows_below]
    r = torch.arange(rows_below, device="cuda")
    strip0 = (n // 64) * 64
    src0 = (strip0 // W) * (R * W) + strip0 % W + b_off         # source row of the strip's first column
    owned = (r[:, None] // 128) >= (src0[None, :] // 128)       # row tiles bi >= bimin[strip]
    rmax = Pm.abs().max(1).values
    scale = torch.outer(rmax, rmax[src]) * K
    bound = 2e-13 * scale + 4e-16 * (C0.t()[:rows_below].abs() + want.abs() + scale)
    err = (got - want).abs()
    assert bool((err[owned] <= bound[owned]).all()), float((err / bound)[owned].max())
    assert bool((got[~owned] == C0.t()[:rows_below][~owned]).all())   # tiles above the diagonal are untouched
    assert bool((Cst.t()[rows_below:] == C0.t()[rows_below:]).all())  # rows beyond M (ldc padding) untouched
    assert float((got - C0.t()[:rows_below]).abs()[owned].max()) > 0      # the update really happened


# ---- fp32 on the tensor cores: the same int8-sliced kernel with 4 slices (28 bits cover the fp32 significand), fp32 C
@pytest.mark.parametrize("n,d,fam", [(4224, 8, ref.SE), (6000, 32, ref.MATERN32)])
def test_fp32_fit_on_tcgen05_matches_fp64_oracle(ag, n, d, fam):
    """auto policy for fp32: n_pad >= 4096 -> 512-wide panels, int8-slice trailing update; logpdf rtol 1e-4 (BASELINE.json)"""
    cfg = ref.make_config("C3", n=n)
    X = np.ascontiguousarray(cfg["X"][:, :d])
    y = cfg["y"]
    ard = np.ascontiguousarray(cfg["k"].ard[:d]) * np.float32(np.sqrt(32.0 / d))
    k64 = ref.KernelSpec(fam, 1.0, ref.T_ARD, ard=ard.astype(np.float64))
    kern = (ag.SqExponentialKernel() if fam == ref.SE else ag.Matern32Kernel()).compose(ag.ARDTransform(ard))
    eng = ag.engine()
    assert eng.get_config().fp32_mode < 0
    lp, post = ag.fit(ag.GP(kern)(ag.RowVecs(X), 0.05), y)
    assert lp.dtype == np.float32
    X64, y64 = X.astype(np.float64), y.astype(np.float64)
    lp_ref = ref.logpdf(k64, cfg["mean"], cfg["noise"], X64, y64)
    assert abs(lp - lp_ref) <= 1e-4 * abs(lp_ref), (lp, lp_ref)
    pr = ref.posterior(k64, cfg["mean"], cfg["noise"], X64, y64)
    Xs = cfg["Xs"][:1024, :d]
    mu, v = ag.mean_and_var(post(ag.RowVecs(Xs), 0.05))     # 1024 columns: the tensor-core forward substitution
    mu_r, v_r = ref.post_mean_and_var(pr, Xs.astype(np.float64), noise_s=cfg["noise"])
    assert np.allclose(mu, mu_r, rtol=2e-3, atol=2e-3) and np.allclose(v, v_r, rtol=2e-3, atol=2e-3)
    # the tensor path really ran: the FFMA path gives different last bits
    eng.set_config(fp32_mode=0)
    lp0, post0 = ag.fit(ag.GP(kern)(ag.RowVecs(X), 0.05), y)
    eng.set_config(fp32_mode=-1)
    assert abs(lp0 - lp_ref) <= 1e-4 * abs(lp_ref)
    assert not np.array_equal(post.data.alpha, post0.data.alpha)


def test_fp64_predict_uses_tensor_forward_substitution(ag):
    """mean_and_var at 1536 test points on an fp64 posterior with n_pad >= 2048: B[below] -= L[below, block] B[block] runs on
    the int8-slice kernel (7 slices, rectangular product); parity with the oracle at fp64 tolerances"""
    n, d = 3000, 6
    cfg = ref.make_config("C2", n=n)
    X = np.ascontiguousarray(cfg["X"][:, :d])
    ks = ref.KernelSpec(ref.SE, 1.0, ref.T_SCALE, scale=1.0 / (0.5 * np.sqrt(d)))
    f = ag.GP(ag.SqExponentialKernel().compose(ag.ScaleTransform(ks.scale)))
    post = ag.posterior(f(ag.RowVecs(X), 0.1), cfg["y"])
    pr = ref.posterior(ks, cfg["mean"], cfg["noise"], X, cfg["y"])
    Xs = np.random.default_rng(4).random((1536, d))
    mu, v = ag.mean_and_var(post, ag.RowVecs(Xs))
    mu_r, v_r = ref.post_mean_and_var(pr, Xs)
    assert np.allclose(mu, mu_r, rtol=1e-7, atol=1e-8) and np.allclose(v, v_r, rtol=1e-6, atol=1e-9)
