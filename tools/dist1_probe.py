"""Drive the DISTRIBUTED fit path on ONE GPU (a 1-rank NCCL communicator) in host-pointer and device-pointer mode and
print the library's phase timings -- to see whether an e2e-only slowdown of the "gram" phase seen at several ranks
is a property of the path or of several processes sharing a host.
Usage: python tools/dist1_probe.py N D [reps]"""
import ctypes as C
import importlib.util
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("agp_cabi", os.path.join(ROOT, "abstractgps.jl_b200", "_cabi.py"))
cabi = importlib.util.module_from_spec(spec)
spec.loader.exec_module(cabi)
N, D = int(sys.argv[1]), int(sys.argv[2])
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 4
for name in ("libcudart.so.12", "libcudart.so", "/usr/local/cuda/lib64/libcudart.so"):
    try:
        rt = C.CDLL(name, mode=C.RTLD_GLOBAL)
        break
    except OSError:
        continue
L = C.CDLL(cabi.LIB_PATH, mode=C.RTLD_GLOBAL)
for name, (res, args) in cabi.SIGNATURES.items():
    fn = getattr(L, name)
    fn.restype, fn.argtypes = res, args
rt.cudaMalloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
rt.cudaHostRegister.argtypes = [C.c_void_p, C.c_size_t, C.c_uint]
idbuf = np.zeros(128, dtype=np.uint8)
assert L.agp_nccl_unique_id(idbuf.ctypes.data) == 0
h = C.c_void_p()
assert L.agp_init_dist(C.byref(h), 0, 0, 1, 1, 1, idbuf.ctypes.data, None) == 0
rng = np.random.default_rng(0)
X = rng.random((N, D))
y = np.sin(2 * np.pi * X.mean(1)) + 0.3 * rng.standard_normal(N)
alpha = np.zeros(N)
for a in (X, y, alpha):
    rt.cudaHostRegister(a.ctypes.data, a.nbytes, 0)  # pinned, like bench.py's e2e arm
ks = cabi.agp_kernel(0, 1, 1.0, 1.0 / (0.5 * np.sqrt(D)), 0.0, None)
ms, ns = cabi.agp_mean(0, 0.0, None), cabi.agp_noise(0, 0.1, None)
lp = np.zeros(1)
dX, dy, da = C.c_void_p(), C.c_void_p(), C.c_void_p()
rt.cudaMalloc(C.byref(dX), X.nbytes); rt.cudaMalloc(C.byref(dy), y.nbytes); rt.cudaMalloc(C.byref(da), alpha.nbytes)
rt.cudaMemcpy(dX, X.ctypes.data, X.nbytes, 1); rt.cudaMemcpy(dy, y.ctypes.data, y.nbytes, 1)
keys = ["total", "h2d", "gram", "cholesky", "solves", "d2h", "predict", "trailing"]
for mode, (xp, yp, ap) in (("device", (dX, dy, da)), ("host", (X.ctypes.data, y.ctypes.data, alpha.ctypes.data)), ("device", (dX, dy, da)), ("host", (X.ctypes.data, y.ctypes.data, alpha.ctypes.data))):
    L.agp_set_memspace(h, 1 if mode == "device" else 0)
    for it in range(reps):
        t0 = time.perf_counter()
        rc = L.agp_fit(h, cabi.AGP_F64, C.byref(ks), C.byref(ms), C.byref(ns), cabi.AGP_POINT_MAJOR, xp, N, D, yp, 1, lp.ctypes.data, ap, None)
        wall = (time.perf_counter() - t0) * 1e3
        assert rc == 0, L.agp_last_error(h).decode()
        tm = (C.c_double * 8)()
        L.agp_last_timings(h, tm, 8)
        print(mode, it, "wall %.1f" % wall, {k: round(tm[i], 2) for i, k in enumerate(keys[:6])}, "logpdf %.10g" % lp[0], flush=True)
