"""Measure the error of agp_post_pred_logpdf_grad on fp32 handles against the fp64 NumPy model (tests/pred_logpdf_grad_ref.py,
evaluated on the fp32-rounded inputs), with the fp64 handle's error beside it:
  1. a sweep over cond(C) = 1e2 .. 1e5 (SE with a Scale transform, D = 2, N = 2000, M = 500, S = 4 mixed weights; the
     training noise is set from the largest eigenvalue of K_xx so that cond(C) hits the target);
  2. the Linear kernel at the sizes of tests/test_gpu_pred_logpdf_grad.py::test_matches_model.
Each output is reported as the normwise relative error |g - g*| / |g*| (the kernel gradient as one vector).  The card's
name and power limit are printed first.
Usage: python tools/pred_logpdf_grad_fp32_error.py"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import agp_b200 as ag  # noqa: E402
import composite_ref as cr  # noqa: E402
import pred_logpdf_grad_ref as pr  # noqa: E402
from oracle import agp_ref as ref  # noqa: E402

KEYS = [("y", "y"), ("x", "x"), ("xs", "xs"), ("Y", "Ys"), ("noise_s", "noise_s_diag")]


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def errors(k, spec, X, y, Xs, Ys, s2, w, dtype):
    p = ag.posterior(ag.GP(0.3, k)(ag.RowVecs(X.astype(dtype)), s2), y.astype(dtype))
    lp, g = ag.posterior_logpdf_grad(p(ag.RowVecs(Xs.astype(dtype)), 0.05), Ys.astype(dtype), lp_bar=w, inputs=True)
    r = lambda a: a.astype(dtype).astype(np.float64)  # noqa: E731
    want = pr.pred_logpdf_grad(spec, ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, float(np.float32(s2)) if dtype == np.float32 else s2),
                               r(X), r(y), r(Xs), ref.MeanSpec(1, 0.3), ref.NoiseSpec(0, 0.05), r(Ys), w)
    kg = [g["variance"]] + ([g["scale"]] if "scale" in g else []) + ([g["linear_c"]] if "linear_c" in g else [])
    kw = [want["grad"][0]] + ([want["grad"][1]] if "scale" in g else []) + ([want["grad"][2]] if "linear_c" in g else [])
    out = {"lp": rel(lp, want["lp"]), "kernel": rel(kg, kw), "noise": rel(g["noise"], want["grad"][3]),
           "mean_c": rel(g["mean_c"], want["grad"][4])}
    for a, b in KEYS:
        out[a] = rel(g[a], np.sum(want[b]) if a == "noise_s" else want[b])
    return out


def line(tag, e32, e64):
    print(tag + "  " + "  ".join("%s %.1e/%.1e" % (key, e32[key], e64[key]) for key in e32), flush=True)


def main():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown (nvidia-smi failed)")
    print("each entry: fp32 / fp64 normwise relative error against the fp64 model")
    rng = np.random.default_rng(5)
    N, M, D, S = 2000, 500, 2, 4
    X, y = rng.uniform(-2, 2, (N, D)), rng.standard_normal(N)
    Xs, Ys = rng.uniform(-2.2, 2.2, (M, D)), rng.standard_normal((M, S))
    w = np.array([1.0, -0.4, 0.0, 1.7])
    k = ag.with_lengthscale(ag.SqExponentialKernel(), 0.8)
    spec = ref.KernelSpec(cr.SE, 1.0, cr.T_SCALE, 1 / 0.8)
    lmax = float(np.linalg.eigvalsh(cr.kernelmatrix(pr.gx.as_composite(spec), X))[-1])
    for cond in (1e2, 1e3, 1e4, 1e5):
        s2 = lmax / (cond - 1.0)
        line("SE cond(C)=%.0e s2=%.2e" % (cond, s2), errors(k, spec, X, y, Xs, Ys, s2, w, np.float32),
             errors(k, spec, X, y, Xs, Ys, s2, w, np.float64))
    for Nl, Ml, Dl, Sl in [(63, 17, 3, 2), (333, 129, 1, 3), (333, 200, 40, 2), (1300, 1000, 3, 130)]:
        rl = np.random.default_rng(Nl)
        Xl, yl = rl.uniform(-2, 2, (Nl, Dl)), rl.standard_normal(Nl)
        Xsl, Ysl = rl.uniform(-2.2, 2.2, (Ml, Dl)), rl.standard_normal((Ml, Sl))
        kl = ag.LinearKernel(c=0.4)
        sl = ref.KernelSpec(cr.LINEAR, 1.0, cr.T_NONE, linear_c=0.4)
        Kl = cr.kernelmatrix(pr.gx.as_composite(sl), Xl)
        cond = (np.linalg.eigvalsh(Kl)[-1] + 0.1) / 0.1
        line("Linear N=%d M=%d D=%d cond(C)=%.1e" % (Nl, Ml, Dl, cond), errors(kl, sl, Xl, yl, Xsl, Ysl, 0.1, None, np.float32),
             errors(kl, sl, Xl, yl, Xsl, Ysl, 0.1, None, np.float64))


if __name__ == "__main__":
    main()
