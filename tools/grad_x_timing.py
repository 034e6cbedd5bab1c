"""Time the input gradient against the hyper-parameter gradient on one GPU: agp_post_logpdf_grad and
agp_post_logpdf_grad_x (hyper-parameters and inputs from one C^-1) alternate on the same handle, each timed with CUDA
events around the call, for
  - SE over an ARD transform at D = 8 and 64, N = 4096 and 16 384, fp64 and fp32;
  - the Mauna Loa composite (D = 1) at N = 16 384, fp64 and fp32.
The card's name and power limit are printed first; the added time is reported as a share of the gradient call.
Usage: python tools/grad_x_timing.py [reps]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import agp_b200 as ag  # noqa: E402


def mauna_loa():
    SE = lambda s, l: s ** 2 * ag.with_lengthscale(ag.SqExponentialKernel(), l)  # noqa: E731
    per = ag.with_lengthscale(ag.PeriodicKernel(r=[0.5]), 1.0)
    rq = ag.with_lengthscale(ag.RationalQuadraticKernel(alpha=np.exp(-1.0)), 1.0)
    return SE(np.exp(4), np.exp(4)) + per * SE(np.exp(1), np.exp(4)) + rq + (SE(np.exp(-2), np.exp(-2)) + np.exp(-4) * ag.WhiteKernel())


def time_case(k, N, D, dtype, reps):
    import torch
    rng = np.random.default_rng(1)
    X = rng.uniform(0, 10, (N, D)).astype(dtype)
    y = np.sin(X).sum(1).astype(dtype)
    post = ag.posterior(ag.GP(k)(ag.RowVecs(X), 0.1 if dtype == np.float64 else 10.0), y)
    eng, h = ag.engine(), post.data.C.h
    g = np.zeros(int(eng.L.agp_post_grad_len(h)))
    gp = g.ctypes.data_as(C.POINTER(C.c_double))
    xg = torch.empty((N, D), dtype=torch.float64 if dtype == np.float64 else torch.float32, device="cuda")
    calls = {"grad": lambda: eng.L.agp_post_logpdf_grad(h, gp, None),
             "grad_x": lambda: eng.L.agp_post_logpdf_grad_x(h, gp, None, 0, C.c_void_p(xg.data_ptr()))}
    eng.set_memspace(ag._cabi.AGP_MEM_DEVICE)  # x_grad_out stays on the device, like a PyTorch caller's
    try:
        for f in calls.values():  # warm-up
            eng.check(f())
        ms = {name: [] for name in calls}
        for _ in range(reps):
            for name, f in calls.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                eng.check(f())
                b.record()
                b.synchronize()
                ms[name].append(a.elapsed_time(b))
    finally:
        eng.set_memspace(ag._cabi.AGP_MEM_HOST)
    return float(np.median(ms["grad"])), float(np.median(ms["grad_x"]))


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown (nvidia-smi failed)")
    cases = []
    for dtype in (np.float64, np.float32):
        for N in (4096, 16384):
            for D in (8, 64):
                v = np.random.default_rng(D).uniform(0.2, 0.6, D) / np.sqrt(D)
                cases.append(("SE/ARD", ag.SqExponentialKernel().compose(ag.ARDTransform(v)), N, D, dtype))
        cases.append(("mauna-loa composite", mauna_loa(), 16384, 1, dtype))
    for name, k, N, D, dtype in cases:
        t0, t1 = time_case(k, N, D, dtype, reps)
        print("%-8s N=%6d D=%3d %-20s grad %9.2f ms  grad_x %9.2f ms  added %7.2f ms = %5.1f %% of grad"
              % (np.dtype(dtype).name, N, D, name, t0, t1, t1 - t0, 100 * (t1 - t0) / t0), flush=True)


if __name__ == "__main__":
    main()
