"""Measure the error of agp_post_rand_grad on fp32 handles against the fp64 NumPy model (tests/post_rand_grad_ref.py,
evaluated on the fp32-rounded inputs), with the fp64 handle's error beside it, as cond(C) and cond(Sigma) grow: SE with a
Scale transform, D = 2, N = 2000, M = 500, S = 16; cond(C) is set by the training noise from the largest eigenvalue of
K_xx (test noise 0.05), then cond(Sigma) by the test noise at cond(C) = 1e3.  Each output is reported as the normwise
relative error |g - g*| / |g*| (the kernel gradient as one vector).  The card's name and power limit are printed first.
Usage: python tools/post_rand_grad_fp32_error.py"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import agp_b200 as ag  # noqa: E402
import composite_ref as cr  # noqa: E402
import grad_x_ref as gx  # noqa: E402
import post_rand_grad_ref as prr  # noqa: E402
from oracle import agp_ref as ref  # noqa: E402

KEYS = [("out", "out"), ("y", "y"), ("x", "x"), ("xs", "xs"), ("Z", "Z"), ("noise_s", "noise_s_diag")]


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def errors(k, spec, X, y, Xs, Z, Ob, s2, s2s, dtype):
    r = lambda a: np.asarray(a).astype(dtype).astype(np.float64)  # noqa: E731
    p = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X.astype(dtype)), s2), y.astype(dtype))
    out, g = ag.posterior_rand_grad(p(ag.RowVecs(Xs.astype(dtype)), s2s), Z.astype(dtype), Ob.astype(dtype), inputs=True)
    g["out"] = out
    want = prr.post_rand_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, float(r(s2))), r(X), r(y), r(Xs), ref.MeanSpec(1, 0.3),
                              ref.NoiseSpec(0, float(r(s2s))), r(Z), r(Ob))
    res = {"kernel": rel([g["variance"], g["scale"]], want["grad"][:2]), "noise": rel(g["noise"], want["grad"][3]),
           "mean_c": rel(g["mean_c"], want["grad"][4])}
    for a, b in KEYS:
        res[a] = rel(g[a], np.sum(want[b]) if a == "noise_s" else want[b])
    return res


def line(tag, e32, e64):
    print(tag + "  " + "  ".join("%s %.1e/%.1e" % (key, e32[key], e64[key]) for key in e32), flush=True)


def main():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown (nvidia-smi failed)")
    print("each entry: fp32 / fp64 normwise relative error against the fp64 model")
    rng = np.random.default_rng(5)
    N, M, D, S = 2000, 500, 2, 16
    X, y = rng.uniform(-2, 2, (N, D)), rng.standard_normal(N)
    Xs, Z, Ob = rng.uniform(-2.2, 2.2, (M, D)), rng.standard_normal((M, S)), rng.standard_normal((M, S))
    k = 1.3 * ag.with_lengthscale(ag.SqExponentialKernel(), 0.8)
    spec = ref.KernelSpec(cr.SE, 1.3, cr.T_SCALE, 1 / 0.8)
    kc = gx.as_composite(spec)
    lmax = float(np.linalg.eigvalsh(cr.kernelmatrix(kc, X))[-1])
    for cond in (1e2, 1e3, 1e4, 1e5):
        s2 = lmax / (cond - 1.0)
        line("cond(C)=%.0e s2=%.2e" % (cond, s2), errors(k, spec, X, y, Xs, Z, Ob, s2, 0.05, np.float32),
             errors(k, spec, X, y, Xs, Z, Ob, s2, 0.05, np.float64))
    s2 = lmax / (1e3 - 1.0)
    for s2s in (1e-1, 1e-2, 1e-3, 1e-4):
        Kxs = cr.kernelmatrix(kc, X, Xs)
        Sig = cr.kernelmatrix(kc, Xs) - Kxs.T @ np.linalg.solve(cr.kernelmatrix(kc, X) + s2 * np.eye(N), Kxs) + s2s * np.eye(M)
        ev = np.linalg.eigvalsh(Sig)
        line("cond(C)=1e+03 cond(Sigma)=%.1e s2*=%.0e" % (ev[-1] / ev[0], s2s),
             errors(k, spec, X, y, Xs, Z, Ob, s2, s2s, np.float32), errors(k, spec, X, y, Xs, Z, Ob, s2, s2s, np.float64))


if __name__ == "__main__":
    main()
