"""The fp64 fit with 1024-wide outer panels (two-level: the first half's update of the second half runs on the eight-bit
kernel, see engine.cu factor_outer_panel) against the fp64 oracle and against the same fit with 512-wide panels, at
sizes where the int8-slice path runs, ragged ones and ones whose last outer panel is partial; a failing pivot in the
second half of a 1024 panel; and a repeated fit on one engine, which must return the same bits."""
import numpy as np
import pytest
import scipy.linalg as sla

pytestmark = pytest.mark.gpu

LS, NOISE, D = 1.5, 0.1, 8


@pytest.fixture
def panel_width(ag):
    eng = ag.engine()
    old = eng.get_config().tile_nb

    def use(nb):
        eng.set_config(tile_nb=nb)

    yield use
    eng.set_config(tile_nb=old)


def _problem(n, seed):
    rng = np.random.default_rng(seed)
    return rng.random((n, D)) * 2.0, rng.standard_normal(n)


def _fx(ag, X, noise=NOISE):
    return ag.GP(ag.with_lengthscale(ag.SqExponentialKernel(), LS))(ag.RowVecs(X), noise)


def _oracle(ref, X, y):
    ks = ref.KernelSpec(ref.SE, 1.0, ref.T_SCALE, 1.0 / LS)
    A = ref.kernelmatrix(ks, X)
    A[np.diag_indices_from(A)] += NOISE
    c = sla.cho_factor(A, lower=True, overwrite_a=True, check_finite=False)
    alpha = sla.cho_solve(c, y, check_finite=False)
    logdet = 2.0 * np.sum(np.log(np.diag(c[0])))
    return -0.5 * (y @ alpha + logdet + len(y) * np.log(2 * np.pi)), alpha


def _fit(ag, X, y):
    lp, post = ag.fit(_fx(ag, X), y)
    return lp, np.array(post.data.alpha, copy=True)


@pytest.mark.parametrize("n", [8192 + 37, 12288, 16384 + 300])
def test_fit_1024_panels(ag, ref, panel_width, n):
    """12 288 fills whole 1024 panels; 8229 and 16 684 end on a partial one (1 and 3 inner blocks)"""
    X, y = _problem(n, n)
    panel_width(1024)
    lp, alpha = _fit(ag, X, y)
    lp2, alpha2 = _fit(ag, X, y)
    assert lp == lp2 and alpha.tobytes() == alpha2.tobytes()  # deterministic from call to call
    panel_width(512)
    lp512, alpha512 = _fit(ag, X, y)
    lp_ref, alpha_ref = _oracle(ref, X, y)
    sc = np.abs(alpha_ref).max()
    for l_, a_ in ((lp, alpha), (lp512, alpha512)):
        assert abs(l_ - lp_ref) <= 1e-8 * abs(lp_ref), (l_, lp_ref)
        assert np.max(np.abs(a_ - alpha_ref)) <= 1e-8 * sc
    assert abs(lp - lp512) <= 1e-8 * abs(lp512)
    assert np.max(np.abs(alpha - alpha512)) <= 1e-8 * np.abs(alpha512).max()


@pytest.mark.parametrize("p", [700, 2048 + 1000])
def test_first_failing_pivot_in_second_half(ag, panel_width, p):
    """a negative noise at point p makes pivot p (0-based) the first that fails: every earlier leading block is the SPD
    kernel matrix plus 0.1 I.  p lies in the second half of the first and of the third 1024 panel"""
    n = 12288 + 64
    X, y = _problem(n, 5)
    noise = np.full(n, NOISE)
    noise[p] = -10.0
    panel_width(1024)
    with pytest.raises(ag.PosDefException) as ei:
        ag.logpdf(_fx(ag, X, noise), y)
    assert ei.value.info == p + 1
    lp, _ = _fit(ag, X[:9000], y[:9000])  # the engine stays usable
    assert np.isfinite(lp)


@pytest.mark.parametrize("n,nb", [(32768 - 128, 512), (32768, 1024)])
def test_automatic_width(ag, panel_width, n, nb):
    """the automatic fp64 width: 512 below n_pad = 32 768, 1024 from there (the same bits as the explicit width)"""
    X, y = _problem(n, 7)
    panel_width(0)
    lp, alpha = _fit(ag, X, y)
    panel_width(nb)
    lp_nb, alpha_nb = _fit(ag, X, y)
    assert lp == lp_nb and alpha.tobytes() == alpha_nb.tobytes()
