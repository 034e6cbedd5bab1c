"""Time the gradient of the held-out log-likelihood on one GPU: agp_post_logpdf (the value alone),
agp_post_logpdf_grad_x (the training logpdf's gradient) and agp_post_pred_logpdf_grad (every output requested, one
target column, lp_bar NULL) alternate on one handle, each timed with CUDA events around the C ABI call (host inputs and
outputs), for fp64 and fp32 at N = 16 384 training points with M = 1024 and 4096 test points.  Two priors: SE over an
ARD transform at D = 8, and the Mauna Loa composite (SE + Periodic * SE + RQ + SE + White, Scale transforms) at D = 1.
Scalar noises, a constant mean.  The card's name and power limit are printed first.
Usage: python tools/pred_logpdf_grad_timing.py [reps]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import agp_b200 as ag  # noqa: E402


def prior(name, D, rng):
    if name == "se_ard":
        return ag.SqExponentialKernel().compose(ag.ARDTransform(rng.uniform(0.5, 1.5, D)))
    se = lambda ls: ag.with_lengthscale(ag.SqExponentialKernel(), ls)  # noqa: E731
    return (1.4 * se(0.5) + 0.8 * (ag.with_lengthscale(ag.PeriodicKernel(r=[0.7]), 0.9) * se(0.4))
            + 0.5 * ag.with_lengthscale(ag.RationalQuadraticKernel(alpha=1.3), 0.8) + 0.1 * se(2.0) + 0.04 * ag.WhiteKernel())


def time_case(name, N, M, dtype, reps):
    import torch
    cabi = ag._cabi
    eng = ag.engine()
    D = 8 if name == "se_ard" else 1
    rng = np.random.default_rng(3)
    X = np.ascontiguousarray(rng.uniform(-1, 1, (N, D)).astype(dtype))
    Xs = np.ascontiguousarray(rng.uniform(-1.1, 1.1, (M, D)).astype(dtype))
    y = rng.standard_normal(N).astype(dtype)
    Ys = np.asfortranarray(rng.standard_normal((M, 1)).astype(dtype))
    k = prior(name, D, rng)
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)
    h = post.data.C.h
    keep = []
    ms = ag.api._mean_struct(post.prior.mean.spec(ag.api._Points(ag.RowVecs(Xs)), dtype), keep)
    ns = cabi.agp_noise(0, 0.05, None)
    g = np.zeros(int(eng.L.agp_post_grad_len(h)))
    gp = g.ctypes.data_as(C.POINTER(C.c_double))
    e = lambda *s: np.empty(s, dtype=dtype)  # noqa: E731
    lp, nd, yb, xg, nsd, ysb, xsg = e(1), e(N), e(N), e(N, D), e(M), e(M, 1), e(M, D)
    P = cabi.ptr
    calls = {
        "logpdf": lambda: eng.L.agp_post_logpdf(h, 0, P(Xs), M, C.byref(ms), C.byref(ns), P(Ys), 1, P(lp)),
        "grad_x": lambda: eng.L.agp_post_logpdf_grad_x(h, gp, P(nd), 0, P(xg)),
        "pred_grad": lambda: eng.L.agp_post_pred_logpdf_grad(h, 0, P(Xs), M, C.byref(ms), C.byref(ns), P(Ys), 1, None, P(lp), gp,
                                                             P(nd), None, P(yb), P(xg), P(nsd), None, P(ysb), P(xsg)),
    }
    for fn in calls.values():  # warm-up
        eng.check(fn())
    ms_ = {n: [] for n in calls}
    for _ in range(reps):
        for n, fn in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            eng.check(fn())
            b.record()
            b.synchronize()
            ms_[n].append(a.elapsed_time(b))
    return {n: float(np.median(v)) for n, v in ms_.items()}


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown (nvidia-smi failed)")
    N = 16384
    for name in ("se_ard", "mauna_loa"):
        for dtype in (np.float64, np.float32):
            for M in (1024, 4096):
                t = time_case(name, N, M, dtype, reps)
                print("%-9s %-8s N=%6d M=%5d reps=%d  post_logpdf %8.1f ms  logpdf_grad_x %8.1f ms  pred_logpdf_grad %8.1f ms"
                      % (name, np.dtype(dtype).name, N, M, reps, t["logpdf"], t["grad_x"], t["pred_grad"]), flush=True)


if __name__ == "__main__":
    main()
