"""int8-sliced (Ozaki) fp64 trailing update (wgmma) vs. a float64 reference computed with torch on the
same device (a floating-point kernel, so the reference is fp64 matmul; the exact-integer part of the
scheme is additionally checked on integer-valued inputs, where the result must be bit-exact)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _run(ag, M, N, K, S, lower, seed=0, integer=False):
    import torch
    eng = ag.engine()
    g = torch.Generator(device="cuda").manual_seed(seed)
    if integer:
        P = torch.randint(-60, 61, (K, M), generator=g, device="cuda").to(torch.float64).t()  # column-major M x K view
    else:
        P = (torch.rand((K, M), generator=g, device="cuda", dtype=torch.float64) * 2 - 1).t()
        P = P * torch.logspace(-3, 2, M, device="cuda", dtype=torch.float64)[:, None]  # very different row scales
    lda = M
    Cm = torch.rand((N, M + 5), generator=g, device="cuda", dtype=torch.float64).t()  # column-major, ldc = M + 5
    ldc = M + 5
    C0 = Cm.clone()
    Pc = P.t().contiguous()      # storage of the column-major M x K matrix
    Cc = Cm.t().contiguous()     # storage of the column-major (M+5) x N matrix
    torch.cuda.synchronize()  # the library works on its own stream: device inputs must be complete before the call
    rc = eng.L.agp_debug_ozaki_syrk(eng.h, C.c_void_p(Cc.data_ptr()), ldc, C.c_void_p(Pc.data_ptr()), lda, M, N, K, S, int(lower))
    eng.check(rc)
    got = Cc.t()[:M, :N]
    want = C0[:M, :N] - P @ P[:N].t()
    return got.cpu().numpy(), want.cpu().numpy(), C0[:M, :N].cpu().numpy(), (P.abs().max(1).values).cpu().numpy()


@pytest.mark.parametrize("M,N,K,S", [(128, 64, 64, 8), (256, 256, 128, 8), (384, 320, 256, 7), (1000, 704, 256, 8), (640, 640, 512, 6)])
def test_ozaki_syrk_matches_fp64(ag, M, N, K, S):
    got, want, c0, rmax = _run(ag, M, N, K, S, lower=False)
    # error model: slicing truncation is relative to the row-scale products (2^-7S), plus the fp64
    # rounding of C itself and of the reference matmul
    scale = np.outer(rmax, rmax[:N]) * K
    tol = {8: 1e-15, 7: 2e-13, 6: 3e-11}[S]
    bound = tol * scale + 4e-16 * (np.abs(c0) + np.abs(want) + scale)
    assert np.all(np.abs(got - want) <= bound), float((np.abs(got - want) / bound).max())


def test_ozaki_exact_on_integers(ag):
    got, want, _, _ = _run(ag, 256, 256, 128, 8, lower=False, integer=True)
    assert np.array_equal(got, want)  # every product and sum is exact in int32 / fp64


def test_ozaki_lower_only_leaves_upper_tiles(ag):
    got, want, c0, _ = _run(ag, 512, 512, 128, 8, lower=True)
    i, j = np.indices(got.shape)
    low = (j // 64) * 64 < (i // 128) * 128 + 128   # tiles the kernel owns
    assert np.allclose(got[low], want[low], rtol=0, atol=1e-9)
    assert np.array_equal(got[~low], c0[~low])       # tiles entirely above the diagonal are untouched


@pytest.mark.parametrize("N,K,S", [(128, 128, 7), (1024, 256, 7), (2048, 512, 8), (2176, 512, 6)])
def test_ozaki_persistent_lower_with_border(ag, N, K, S):
    """the persistent (v2) kernel on the shape the Cholesky uses: M = N + 128 border rows, lower tiles only"""
    got, want, c0, rmax = _run(ag, N + 128, N, K, S, lower=True, seed=3)
    i, j = np.indices(got.shape)
    low = (j // 64) * 64 < (i // 128) * 128 + 128
    scale = np.outer(rmax, rmax[:N]) * K
    tol = {8: 1e-15, 7: 2e-13, 6: 3e-11}[S]
    bound = tol * scale + 4e-16 * (np.abs(c0) + np.abs(want) + scale)
    assert np.all(np.abs(got - want)[low] <= bound[low]), float((np.abs(got - want) / bound)[low].max())
    assert np.array_equal(got[~low], c0[~low])


# ---- generalised int8-slice path: fp32 / fp64 operands in either storage order, fp32 / fp64 output, rectangular
# products with two operands in one slice workspace, accumulation sign -- the building block of the fp32 factorisation,
# of the multi-RHS forward substitution (C.U' \ X, /root/reference/src/util/common_covmat_ops.jl:54,90) and of the VFE stream
@pytest.mark.parametrize("M,N,K,S,cdt,adt,bdt,akm,bkm,sign", [
    (256, 128, 128, 4, "f32", "f32", "f32", 0, 0, -1.0),
    (1000, 384, 512, 4, "f32", "f32", "f32", 0, 1, -1.0),
    (640, 640, 256, 3, "f32", "f32", "f32", 1, 0, 1.0),
    (900, 256, 2048, 4, "f32", "f32", "f32", 0, 1, 1.0),
    (512, 512, 512, 7, "f64", "f64", "f64", 0, 1, -1.0),
    (1300, 256, 256, 7, "f64", "f64", "f64", 1, 1, 1.0),
    (384, 128, 4096, 5, "f64", "f32", "f32", 0, 0, 1.0),
])
def test_ozaki_general_product(ag, M, N, K, S, cdt, adt, bdt, akm, bkm, sign):
    import torch
    eng = ag.engine()
    td = {"f32": torch.float32, "f64": torch.float64}
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = (torch.rand((M, K), generator=g, device="cuda", dtype=torch.float64) * 2 - 1) * torch.logspace(-2, 2, M, device="cuda", dtype=torch.float64)[:, None]
    B = (torch.rand((N, K), generator=g, device="cuda", dtype=torch.float64) * 2 - 1) * torch.logspace(-1, 1, N, device="cuda", dtype=torch.float64)[:, None]
    A, B = A.to(td[adt]), B.to(td[bdt])
    C0 = torch.rand((N, M + 3), generator=g, device="cuda", dtype=torch.float64).to(td[cdt])  # storage of col-major (M+3) x N
    Cst = C0.clone()
    # storage: row-contiguous operand = col-major M x K = tensor [K, M]; k-major = tensor [M, K]
    Ast = A.contiguous() if akm else A.t().contiguous()
    Bst = B.contiguous() if bkm else B.t().contiguous()
    torch.cuda.synchronize()
    rc = eng.L.agp_debug_ozaki_gemm(eng.h, C.c_void_p(Cst.data_ptr()), int(cdt == "f32"), M + 3, C.c_void_p(Ast.data_ptr()),
                                    int(adt == "f32"), akm, K if akm else M, M, C.c_void_p(Bst.data_ptr()), int(bdt == "f32"), bkm,
                                    K if bkm else N, N, K, S, sign)
    eng.check(rc)
    want = C0.t()[:M].double() + sign * (A.double() @ B.double().t())
    got = Cst.t()[:M].double()
    scale = torch.outer(A.double().abs().max(1).values, B.double().abs().max(1).values) * K
    eps_c = 6e-8 if cdt == "f32" else 1.2e-16
    trunc = {3: 2.0 ** -19, 4: 2.0 ** -26, 5: 2.0 ** -33, 7: 2.0 ** -47}[S]
    bound = trunc * scale + 2 * eps_c * (want.abs() + C0.t()[:M].double().abs() + scale * (1e-9 if cdt == "f64" else 0) + 1e-30)
    err = (got - want).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    assert bool((Cst.t()[M:] == C0.t()[M:]).all())


@pytest.mark.parametrize("N,K,S", [(512, 512, 4), (1152, 1024, 3)])
def test_ozaki_fp32_syrk_lower(ag, N, K, S):
    """the fp32 trailing update: lower tiles of C -= P P' with M = N + 128 border rows, fp32 panel and fp32 C"""
    import torch
    eng = ag.engine()
    M = N + 128
    g = torch.Generator(device="cuda").manual_seed(7)
    P = ((torch.rand((M, K), generator=g, device="cuda", dtype=torch.float64) * 2 - 1)).float()
    C0 = torch.rand((N, M), generator=g, device="cuda", dtype=torch.float32)
    Cst = C0.clone()
    Pst = P.t().contiguous()
    torch.cuda.synchronize()
    eng.check(eng.L.agp_debug_ozaki_gemm(eng.h, C.c_void_p(Cst.data_ptr()), 1, M, C.c_void_p(Pst.data_ptr()), 1, 0, M, M, None, 0, 0, 0,
                                         N, K, S, -1.0))
    want = C0.t().double() - P.double() @ P.double()[:N].t()
    got = Cst.t().double()
    i, j = np.indices((M, N))
    low = torch.from_numpy((j // 64) * 64 < (i // 128) * 128 + 128).cuda()
    tol = {3: 2.0 ** -19, 4: 2.0 ** -26}[S] * K + 2e-7 * (want.abs() + 1)
    assert bool(((got - want).abs()[low] <= tol[low]).all()), float(((got - want).abs() / tol)[low].max())
    assert bool((got[~low] == C0.t().double()[~low]).all())
