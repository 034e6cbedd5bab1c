"""Time the gradient of logpdf(fx, Y) for a matrix Y on one GPU: agp_post_logpdf_grad_x and agp_post_logpdf_grad_cols
(every output requested, lp_bar NULL) alternate on one handle, each timed with CUDA events around the C ABI call (host
inputs and outputs), for fp64 and fp32 at N = 4096 and 16 384 with S = 1, 128 and 1024 columns.  SE over an ARD
transform, D = 8, scalar noise, a constant mean.  The card's name and power limit are printed first.
Usage: python tools/logpdf_grad_cols_timing.py [reps]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import agp_b200 as ag  # noqa: E402


def time_case(N, S, dtype, reps, D=8):
    import torch
    cabi = ag._cabi
    eng = ag.engine()
    rng = np.random.default_rng(3)
    X = np.ascontiguousarray(rng.uniform(-1, 1, (N, D)).astype(dtype))
    Y = np.asfortranarray(rng.standard_normal((N, S)).astype(dtype))
    k = ag.SqExponentialKernel().compose(ag.ARDTransform(rng.uniform(0.5, 1.5, D)))
    post = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X), 0.1), Y[:, 0].copy())
    h = post.data.C.h
    g = np.zeros(5 + D)
    gp = g.ctypes.data_as(C.POINTER(C.c_double))
    nd, md, xg = np.empty(N, dtype=dtype), np.empty(N, dtype=dtype), np.empty((N, D), dtype=dtype)
    yb = np.empty((N, S), dtype=dtype, order="F")
    calls = {
        "grad_x": lambda: eng.L.agp_post_logpdf_grad_x(h, gp, cabi.ptr(nd), 0, cabi.ptr(xg)),
        "grad_cols": lambda: eng.L.agp_post_logpdf_grad_cols(h, None, cabi.ptr(Y), S, None, gp, cabi.ptr(nd), cabi.ptr(md), 0,
                                                             cabi.ptr(xg), cabi.ptr(yb)),
    }
    for fn in calls.values():  # warm-up
        eng.check(fn())
    ms_ = {name: [] for name in calls}
    for _ in range(reps):
        for name, fn in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            eng.check(fn())
            b.record()
            b.synchronize()
            ms_[name].append(a.elapsed_time(b))
    return {name: float(np.median(v)) for name, v in ms_.items()}


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown (nvidia-smi failed)")
    for dtype in (np.float64, np.float32):
        for N in (4096, 16384):
            for S in (1, 128, 1024):
                t = time_case(N, S, dtype, reps)
                print("%-8s N=%6d S=%5d reps=%d  logpdf_grad_x %9.1f ms  logpdf_grad_cols %9.1f ms  added %+8.1f ms"
                      % (np.dtype(dtype).name, N, S, reps, t["grad_x"], t["grad_cols"], t["grad_cols"] - t["grad_x"]),
                      flush=True)


if __name__ == "__main__":
    main()
