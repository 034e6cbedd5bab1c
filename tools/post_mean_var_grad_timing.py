"""Time the pullback of mean_and_var over an exact posterior on one GPU: agp_post_mean_var (the values alone),
agp_post_mean_var_grad with only xs_grad_out (the test-side-only call an optimiser over x* makes),
agp_post_mean_var_grad with every output, and agp_post_rand_grad at S = 1 with every output alternate on one handle, each
timed with CUDA events around the C ABI call (host inputs and outputs), for fp64 and fp32 at N = 4096 and 16 384
training points with M = 1, 64, 1024 and 4096 test points.  The prior is SE over an ARD transform at D = 8 with a scalar
noise and a constant mean.  The card's name and power limit are printed first.
Usage: python tools/post_mean_var_grad_timing.py [reps] [N ...]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import agp_b200 as ag  # noqa: E402

D = 8


def handle(N, dtype):
    rng = np.random.default_rng(3)
    X = np.ascontiguousarray(rng.uniform(-1, 1, (N, D)).astype(dtype))
    y = rng.standard_normal(N).astype(dtype)
    k = ag.SqExponentialKernel().compose(ag.ARDTransform(rng.uniform(0.5, 1.5, D)))
    return ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), y)


def time_case(post, N, M, dtype, reps):
    import torch
    cabi = ag._cabi
    eng = ag.engine()
    rng = np.random.default_rng(5)
    Xs = np.ascontiguousarray(rng.uniform(-1.1, 1.1, (M, D)).astype(dtype))
    mb, vb = rng.standard_normal(M).astype(dtype), rng.standard_normal(M).astype(dtype)
    Z = np.asfortranarray(rng.standard_normal((M, 1)).astype(dtype))
    Ob = np.asfortranarray(rng.standard_normal((M, 1)).astype(dtype))
    h = post.data.C.h
    keep = []
    ms = ag.api._mean_struct(post.prior.mean.spec(ag.api._Points(ag.RowVecs(Xs)), dtype), keep)
    ns = cabi.agp_noise(0, 0.05, None)
    g = np.zeros(int(eng.L.agp_post_grad_len(h)))
    gp = g.ctypes.data_as(C.POINTER(C.c_double))
    e = lambda *s: np.empty(s, dtype=dtype)  # noqa: E731
    mu, var, nd, yb, xg, nsd, zb, xsg = e(M), e(M), e(N), e(N), e(N, D), e(M), e(M, 1), e(M, D)
    P = cabi.ptr
    calls = {
        "mean_var": lambda: eng.L.agp_post_mean_var(h, 0, P(Xs), M, C.byref(ms), C.byref(ns), P(mu), P(var)),
        "grad_xs": lambda: eng.L.agp_post_mean_var_grad(h, 0, P(Xs), M, P(mb), P(vb), None, None, None, None, None, P(xsg)),
        "grad_all": lambda: eng.L.agp_post_mean_var_grad(h, 0, P(Xs), M, P(mb), P(vb), gp, P(nd), None, P(yb), P(xg),
                                                         P(xsg)),
        "rand_grad": lambda: eng.L.agp_post_rand_grad(h, 0, P(Xs), M, C.byref(ms), C.byref(ns), P(Z), 1, P(Ob), gp, P(nd),
                                                      None, P(yb), P(xg), P(nsd), None, P(zb), P(xsg)),
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
    Ns = [int(a) for a in sys.argv[2:]] or [4096, 16384]
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown (nvidia-smi failed)")
    for dtype in (np.float64, np.float32):
        for N in Ns:
            post = handle(N, dtype)
            for M in (1, 64, 1024, 4096):
                t = time_case(post, N, M, dtype, reps)
                print("%-8s N=%6d M=%5d reps=%d  post_mean_var %8.2f ms  grad xs only %8.2f ms  grad all %8.2f ms  "
                      "post_rand_grad S=1 %8.2f ms" % (np.dtype(dtype).name, N, M, reps, t["mean_var"], t["grad_xs"],
                                                       t["grad_all"], t["rand_grad"]), flush=True)
            del post


if __name__ == "__main__":
    main()
