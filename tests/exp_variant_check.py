"""Helper for tests/test_gpu_variants_grad_vfecov.py (run as a subprocess so that a device trap in an unvalidated kernel
cannot poison the pytest process): runs the int8-slice SYRK with the default (persistent) launch and with the given
environment switches on the same inputs and prints the largest difference.
Usage: python tests/exp_variant_check.py N K S AGP_OZAKI_CHUNK_TEST=4 [AGP_OZAKI_EPI=0 ...]"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import agp_b200 as ag
    N, K, S = (int(v) for v in sys.argv[1:4])
    M = N + 128
    eng = ag.engine()
    g = torch.Generator(device="cuda").manual_seed(1)
    P = (torch.rand((K, M), generator=g, device="cuda", dtype=torch.float64) * 2 - 1).t()
    P = P * torch.logspace(-3, 2, M, device="cuda", dtype=torch.float64)[:, None]
    Pc = P.t().contiguous()
    C0 = torch.rand((N, M), generator=g, device="cuda", dtype=torch.float64)
    outs = []
    switches = dict(a.split("=", 1) for a in sys.argv[4:])
    for on in (False, True):
        for k_, v_ in switches.items():
            if on:
                os.environ[k_] = v_
            else:
                os.environ.pop(k_, None)
        Cc = C0.clone()
        torch.cuda.synchronize()  # the library works on its OWN stream: device inputs must be complete before the call
        eng.check(eng.L.agp_debug_ozaki_syrk(eng.h, C.c_void_p(Cc.data_ptr()), M, C.c_void_p(Pc.data_ptr()), M, M, N, K, S, 1))
        torch.cuda.synchronize()
        outs.append(Cc.cpu().numpy())
    d = np.abs(outs[0] - outs[1]).max()
    changed = float(np.abs(outs[1] - C0.cpu().numpy()).max())
    rmax = P.abs().max(1).values.cpu().numpy()
    scale = np.abs(outs[0]) + K * np.outer(rmax[:N], rmax).astype(np.float64)  # storage is N x M (column-major M x N)
    rel = float((np.abs(outs[0] - outs[1]) / scale).max())
    print("MAXDIFF %.3e CHANGED %.3e REL %.3e" % (d, changed, rel))


if __name__ == "__main__":
    main()
