"""Time the input gradient of the elbo against the rest of the gradient on one GPU: approx_log_evidence_grad with
inputs=False (agp_vfe_elbo_grad) and inputs=True (agp_vfe_elbo_grad_x) alternate on the same problem, each timed with
CUDA events around the call (host inputs and outputs, so both include the same uploads), for
  - fp64, N = 100 000, M = 1024 and 4096;
  - fp32, N = 1 000 000, M = 8192 (the C5 shape).
SE over a Scale transform, D = 16, per-point noise.  The card's name and power limit are printed first; the added time is
reported as a share of the gradient call.
Usage: python tools/vfe_grad_x_timing.py [reps]"""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import agp_b200 as ag  # noqa: E402


def time_case(N, M, dtype, reps, D=16):
    import torch
    rng = np.random.default_rng(3)
    X = rng.uniform(-1, 1, (N, D)).astype(dtype)
    y = np.sin(3 * X).sum(1).astype(dtype)
    Z = X[rng.permutation(N)[:M]].copy()
    f = ag.GP(ag.with_lengthscale(ag.SqExponentialKernel(), 2.0))
    fx = f(ag.RowVecs(X), rng.uniform(0.05, 0.2, N).astype(dtype))
    vfe = ag.VFE(f(ag.RowVecs(Z), 1e-6 if dtype == np.float64 else 1e-4))
    calls = {"grad": lambda: ag.approx_log_evidence_grad(vfe, fx, y),
             "grad_x": lambda: ag.approx_log_evidence_grad(vfe, fx, y, inputs=True)}
    for fn in calls.values():  # warm-up
        fn()
    ms = {name: [] for name in calls}
    for _ in range(reps):
        for name, fn in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ms[name].append(a.elapsed_time(b))
    return float(np.median(ms["grad"])), float(np.median(ms["grad_x"]))


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown (nvidia-smi failed)")
    for dtype, N, M in [(np.float64, 100_000, 1024), (np.float64, 100_000, 4096), (np.float32, 1_000_000, 8192)]:
        t0, t1 = time_case(N, M, dtype, reps)
        print("%-8s N=%8d M=%5d  reps=%d  grad %9.1f ms  grad with x %9.1f ms  added %9.1f ms = %6.1f %% of grad"
              % (np.dtype(dtype).name, N, M, reps, t0, t1, t1 - t0, 100 * (t1 - t0) / t0), flush=True)


if __name__ == "__main__":
    main()
