"""Run under torchrun on >= 2 GPUs: the distributed fit (column-cyclic Cholesky + NCCL panel broadcast) must
match the oracle and the single-GPU result.  Prints DIST_OK on rank 0."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import agp_b200 as ag  # noqa: E402
from agp_b200 import _cabi as cabi  # noqa: E402
from agp_b200.dist import init_distributed_engine  # noqa: E402
from oracle import agp_ref as ref  # noqa: E402


def main():
    eng = init_distributed_engine()
    rank = getattr(eng, "rank", 0)
    ok = True
    only_stress = os.environ.get("DIST_CHECK_ONLY_STRESS") == "1"
    for (n, d, dtype, fam) in [] if only_stress else [(300, 3, np.float64, ref.SE), (1537, 8, np.float64, ref.MATERN32), (1000, 4, np.float32, ref.SE),
                               (128, 2, np.float64, ref.SE), (2100, 6, np.float64, ref.MATERN52)]:
        rng = np.random.default_rng(n)
        X = rng.random((n, d)).astype(dtype)
        Y = np.asfortranarray(np.stack([np.sin(X.sum(1)), rng.standard_normal(n)], 1).astype(dtype))
        ksr = ref.KernelSpec(fam, 1.3, ref.T_SCALE, scale=1.0 / (0.5 * np.sqrt(d)))
        ks = cabi.agp_kernel()
        ks.family, ks.transform, ks.variance, ks.scale = fam, 1, 1.3, ksr.scale
        ms = cabi.agp_mean()
        ms.kind, ms.c = 1, 0.25
        ns = cabi.agp_noise()
        ns.kind, ns.s = 0, 0.1
        lp = np.zeros(2, dtype=dtype)
        alpha = np.zeros(n, dtype=dtype)
        post = C.c_void_p()
        rc = eng.L.agp_fit(eng.h, cabi.dtype_code(dtype), C.byref(ks), C.byref(ms), C.byref(ns), cabi.AGP_POINT_MAJOR,
                           cabi.ptr(X), n, d, cabi.ptr(Y), 2, cabi.ptr(lp), cabi.ptr(alpha), C.byref(post))
        eng.check(rc)
        lp_ref = ref.logpdf(ksr, ref.MeanSpec(1, 0.25), ref.NoiseSpec(0, 0.1), X, Y)
        pr = ref.posterior(ksr, ref.MeanSpec(1, 0.25), ref.NoiseSpec(0, 0.1), X, Y[:, 0])
        rt = 1e-8 if dtype == np.float64 else 1e-4
        good = np.allclose(lp, lp_ref, rtol=rt, atol=0 if dtype == np.float64 else 1e-2)
        sc = np.abs(pr["alpha"]).max()
        good &= np.allclose(alpha, pr["alpha"], rtol=1e-6 if dtype == np.float64 else 1e-2,
                            atol=(1e-7 if dtype == np.float64 else 5e-3) * sc)
        # the distributed posterior handle: mean_and_var at M test points (partitioned over the ranks after the factor
        # is gathered), /root/reference/src/exact_gpr_posterior.jl:85-90, and the exported factor U
        M = 257
        Xs = np.random.default_rng(n + 1).random((M, d)).astype(dtype)
        mu, var = np.zeros(M, dtype=dtype), np.zeros(M, dtype=dtype)
        eng.check(eng.L.agp_post_mean_var(post, cabi.AGP_POINT_MAJOR, cabi.ptr(Xs), M, None, C.byref(ns), cabi.ptr(mu), cabi.ptr(var)))
        mu_r, var_r = ref.post_mean_and_var(pr, Xs, noise_s=ref.NoiseSpec(0, 0.1))
        tol = dict(rtol=1e-6, atol=1e-7) if dtype == np.float64 else dict(rtol=5e-3, atol=5e-3)
        good_p = np.allclose(mu, mu_r, **tol) and np.allclose(var, var_r, **tol)
        ld = C.c_double()
        eng.check(eng.L.agp_post_logdet(post, C.byref(ld)))
        good_p &= bool(np.isclose(ld.value, ref.logdet_chol(pr["U"]), rtol=1e-9 if dtype == np.float64 else 1e-4))
        if n <= 1537:
            U = np.zeros((n, n), dtype=dtype, order="F")
            eng.check(eng.L.agp_post_factor_export(post, cabi.ptr(U)))
            good_p &= bool(np.allclose(U, pr["U"], rtol=1e-7 if dtype == np.float64 else 1e-2, atol=1e-9 if dtype == np.float64 else 2e-3))
        eng.L.agp_post_free(post)
        if rank == 0 or not (good and good_p):
            print("[rank %d] n=%d %s fam=%d: logpdf %s ref %s  ok=%s  posterior(mean_and_var, logdet, U) ok=%s  max|dmu|=%.3g max|dvar|=%.3g"
                  % (rank, n, np.dtype(dtype).name, fam, lp, lp_ref, good, good_p, np.abs(mu - mu_r).max(), np.abs(var - var_r).max()), flush=True)
        ok &= bool(good) and bool(good_p)
    # a case large enough for the int8-slice trailing update with the block-cyclic strip table (n_pad >= 8192, W = 512)
    if os.environ.get("DIST_CHECK_LARGE", "1") == "1" and not only_stress:
        n, d = 8704, 8
        cfg = ref.make_config("C4", n=n)
        X = np.ascontiguousarray(cfg["X"][:, :d])
        yv = np.asfortranarray(cfg["y"].reshape(-1, 1))
        ksr = ref.KernelSpec(ref.SE, 1.0, ref.T_SCALE, scale=1.0 / (0.5 * np.sqrt(d)))
        ks = cabi.agp_kernel()
        ks.family, ks.transform, ks.variance, ks.scale = 0, 1, 1.0, ksr.scale
        ns = cabi.agp_noise()
        ns.kind, ns.s = 0, 0.1
        lp = np.zeros(1)
        alpha = np.zeros(n)
        post = C.c_void_p()
        eng.check(eng.L.agp_fit(eng.h, cabi.AGP_F64, C.byref(ks), None, C.byref(ns), cabi.AGP_POINT_MAJOR, cabi.ptr(X), n, d,
                                cabi.ptr(yv), 1, cabi.ptr(lp), cabi.ptr(alpha), C.byref(post)))
        lp_ref = ref.logpdf(ksr, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, yv[:, 0])
        pr = ref.posterior(ksr, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, yv[:, 0])
        good = abs(lp[0] - lp_ref) <= 1e-8 * abs(lp_ref)
        good &= np.allclose(alpha, pr["alpha"], rtol=1e-6, atol=1e-7 * np.abs(pr["alpha"]).max())
        M = 1000
        Xs = np.random.default_rng(3).random((M, d))
        mu, var = np.zeros(M), np.zeros(M)
        eng.check(eng.L.agp_post_mean_var(post, cabi.AGP_POINT_MAJOR, cabi.ptr(Xs), M, None, None, cabi.ptr(mu), cabi.ptr(var)))
        mu_r, var_r = ref.post_mean_and_var(pr, Xs)
        good &= np.allclose(mu, mu_r, rtol=1e-6, atol=1e-7) and np.allclose(var, var_r, rtol=1e-6, atol=1e-8)
        eng.L.agp_post_free(post)
        if rank == 0 or not good:
            print("[rank %d] large n=%d (int8 slices + strip table): logpdf %r ref %r ok=%s" % (rank, n, lp[0], lp_ref, bool(good)), flush=True)
        ok &= bool(good)
    # repeated fits at sizes where every rank owns few outer blocks (n_pad = a small multiple of 512 x ranks): steps are short,
    # so any missing dependency between the main-stream chain and the side-stream rest updates shows up as a wrong logpdf
    # (or a non-PD exit); the result must be identical from run to run
    if os.environ.get("DIST_CHECK_LARGE", "1") == "1":
        sizes = (8192, 6144, 12288)
        if os.environ.get("DIST_CHECK_SIZES"):
            sizes = tuple(int(v) for v in os.environ["DIST_CHECK_SIZES"].split(","))
        for n in sizes:
            d = 8
            cfg = ref.make_config("C4", n=n)
            X = np.ascontiguousarray(cfg["X"][:, :d])
            yv = np.asfortranarray(cfg["y"].reshape(-1, 1))
            ksr = ref.KernelSpec(ref.SE, 1.0, ref.T_SCALE, scale=1.0 / (0.5 * np.sqrt(d)))
            ks = cabi.agp_kernel()
            ks.family, ks.transform, ks.variance, ks.scale = 0, 1, 1.0, ksr.scale
            ns = cabi.agp_noise()
            ns.kind, ns.s = 0, 0.1
            lp_ref = ref.logpdf(ksr, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X, yv[:, 0])
            vals = []
            for rep in range(4):
                lp = np.zeros(1)
                rc = eng.L.agp_fit(eng.h, cabi.AGP_F64, C.byref(ks), None, C.byref(ns), cabi.AGP_POINT_MAJOR, cabi.ptr(X), n, d,
                                   cabi.ptr(yv), 1, cabi.ptr(lp), None, None)
                vals.append((rc, float(lp[0])))
            # (the sqmahal reduction uses floating-point atomics: the last bits may differ from run to run)
            good = all(rc == 0 and abs(v - lp_ref) <= 1e-8 * abs(lp_ref) for rc, v in vals) and \
                max(v for _, v in vals) - min(v for _, v in vals) <= 1e-11 * abs(lp_ref)
            if rank == 0 or not good:
                print("[rank %d] repeat n=%d: %s ref %r ok=%s" % (rank, n, vals, lp_ref, good), flush=True)
            ok &= bool(good)
    # VFE elbo with the data dimension sharded over the ranks (one all-reduce): must match the oracle
    for dtype in () if only_stress else (np.float64, np.float32):
        n, m, d = 3000, 200, 4
        rng = np.random.default_rng(5)
        X = rng.random((n, d)).astype(dtype)
        yv = (np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n)).astype(dtype)
        Z = X[rng.permutation(n)[:m]].copy()
        ksr = ref.KernelSpec(ref.SE, 1.0, ref.T_SCALE, scale=1.0)
        ks = cabi.agp_kernel()
        ks.family, ks.transform, ks.variance, ks.scale = 0, 1, 1.0, 1.0
        ns = cabi.agp_noise()
        ns.kind, ns.s = 0, 0.1
        js = cabi.agp_noise()
        js.kind, js.s = 0, (1e-6 if dtype == np.float64 else 1e-3)
        out = np.zeros(2, dtype=dtype)
        rc = eng.L.agp_vfe_elbo(eng.h, cabi.dtype_code(dtype), C.byref(ks), None, C.byref(ns), cabi.AGP_POINT_MAJOR,
                                cabi.ptr(X), n, d, cabi.ptr(Z), m, C.byref(js), cabi.ptr(yv), cabi.ptr(out[0:1]), cabi.ptr(out[1:2]))
        eng.check(rc)
        el = ref.elbo(ksr, ref.MeanSpec(), ref.NoiseSpec(0, 0.1), X.astype(np.float64), yv.astype(np.float64),
                      Z.astype(np.float64), ref.NoiseSpec(0, js.s))
        good = abs(out[0] - el) <= (1e-8 if dtype == np.float64 else 2e-3) * abs(el)
        if rank == 0 or not good:
            print("[rank %d] vfe %s: elbo %r ref %r ok=%s" % (rank, np.dtype(dtype).name, out[0], el, good), flush=True)
        ok &= bool(good)
    # non-PD must surface on every rank, not hang
    n = 200
    X = np.zeros((n, 1))
    Y = np.zeros((n, 1), order="F")
    ks = cabi.agp_kernel()
    ks.family, ks.transform, ks.variance, ks.scale = 0, 0, 1.0, 1.0
    ns = cabi.agp_noise()
    ns.kind, ns.s = 0, -0.5
    lp = np.zeros(1)
    rc = eng.L.agp_fit(eng.h, cabi.AGP_F64, C.byref(ks), None, C.byref(ns), cabi.AGP_POINT_MAJOR, cabi.ptr(X), n, 1,
                       cabi.ptr(Y), 1, cabi.ptr(lp), None, None)
    if rc != cabi.AGP_ERR_NOT_POSDEF:
        print("[rank %d] non-PD case returned %d instead of AGP_ERR_NOT_POSDEF" % (rank, rc), flush=True)
    ok &= (rc == cabi.AGP_ERR_NOT_POSDEF)
    import torch
    import torch.distributed as dist
    t = torch.tensor([1.0 if ok else 0.0])
    if dist.is_initialized():
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("DIST_OK" if t.item() == 1.0 else "DIST_FAIL", flush=True)
    sys.exit(0 if t.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
