"""Time fits with composite kernels against a plain SE fit on one GPU: the Gram phase (agp_last_timings[2]) and the whole
fit ([0]), for
  - fp64 at N = 16 384 and 65 536: the Mauna Loa prior (D = 1), a 3-term ARD composite (D = 8), and SE at the same N, D;
  - fp32 at N = 16 384: the same three kernels.
The card's name and power limit are read in the same run and printed first.  Noise 0.1 (fp64) or 10 (fp32).  Usage: python tools/composite_timing.py"""
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


def ard3(D):
    rng = np.random.default_rng(0)
    v = lambda: rng.uniform(0.2, 0.6, D)  # noqa: E731
    return (ag.SqExponentialKernel().compose(ag.ARDTransform(v()))
            + 0.5 * ag.Matern52Kernel().compose(ag.ARDTransform(v())) * ag.PeriodicKernel(r=[1.0]).compose(ag.ARDTransform(v()))
            + 0.3 * ag.RationalQuadraticKernel(alpha=1.5).compose(ag.ARDTransform(v())))


def fit_ms(k, N, D, dtype, reps=3):
    rng = np.random.default_rng(1)
    X = rng.uniform(0, 10, (N, D)).astype(dtype)
    y = np.sin(X).sum(1).astype(dtype)
    # fp32 needs more noise for the long-lengthscale terms (variance e^8) to stay positive definite at this N
    fx = ag.GP(k)(ag.RowVecs(X), 0.1 if dtype == np.float64 else 10.0)
    ag.logpdf(fx, y)  # warm-up
    out = []
    for _ in range(reps):
        ag.logpdf(fx, y)
        t = ag.engine().timings()
        out.append((t["gram"], t["total"]))
    return min(out, key=lambda x: x[1])


def main():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown (nvidia-smi failed)")
    rows = []
    for dtype, Ns in ((np.float64, (16384, 65536)), (np.float32, (16384,))):
        for N in Ns:
            for name, k, D in (("mauna-loa composite", mauna_loa(), 1), ("SE", ag.with_lengthscale(ag.SqExponentialKernel(), 2.0), 1),
                               ("3-term ARD composite", ard3(8), 8), ("SE", ag.with_lengthscale(ag.SqExponentialKernel(), 2.0), 8)):
                g, tot = fit_ms(k, N, D, dtype)
                rows.append((np.dtype(dtype).name, N, D, name, g, tot))
                print("%-8s N=%6d D=%d %-22s gram %9.2f ms  fit %9.2f ms  gram share %5.1f %%"
                      % (np.dtype(dtype).name, N, D, name, g, tot, 100 * g / tot), flush=True)


if __name__ == "__main__":
    main()
