"""Six 8-bit slices (ozaki_slices = 6, the default) against seven 7-bit slices (ozaki_slices = 7) on the benchmark's
own problems, alternated in one process on one engine so both formats see the same inputs, card and clocks:
  - C4 (N = 65 536) and C4h (N = 32 768), fp64, D = 64: step time (device-resident, CUDA events, L2 flushed, as
    bench.py), clocks and clock-event reasons during each window, `reps` alternations; then the trailing-kernel time per
    step (profile_kernels = 1, look-ahead off, as bench.py's roofline); logpdf and alpha of the two formats against each
    other, and logpdf against the fp64 oracle on the first 8192 points (bench.py's parity check);
  - C2 and C3 at both settings, which do not run the int8-slice fp64 path, as a control.
The card's name, power limit and maximum SM clock are printed first.  Prints one JSON object per measurement.
Usage: python tools/ozaki8_timing.py [reps]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return {"query": q, "value": r.stdout.strip()}


def window(prob, eng, torch, flush, S, steps):
    """one timed window at ozaki_slices = S (one warm-up step re-slices into the format's workspace)"""
    eng.set_config(ozaki_slices=S)
    sampler = bench.ClockSampler(0)
    sampler.start()
    t, _, _ = bench.timed(prob, torch, flush, True, steps, 1)
    clocks = sampler.stop()
    return {"ms": t["total"], "cholesky_ms": t.get("cholesky"), "clocks": clocks}


def outputs(prob, torch):
    torch.cuda.synchronize()
    return float(prob.lp[0]), prob.alpha_d.cpu().numpy().copy()


def main():
    import torch
    import agp_b200 as ag
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    print(json.dumps({"card": card()}), flush=True)
    eng = ag.engine()
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    cfg0 = eng.get_config()
    for wl, steps in (("C4", 5), ("C4h", 10), ("C2", 20), ("C3", 10)):
        prob = bench.FitProblem(wl, None, eng, torch, dev)
        bench.timed(prob, torch, flush, True, 1, 2)  # first launches of this problem's shapes, untimed
        runs = {6: [], 7: []}
        out = {}
        for _ in range(reps if wl in ("C4", "C4h") else 2):
            for S in (6, 7):
                runs[S].append(window(prob, eng, torch, flush, S, steps))
                out[S] = outputs(prob, torch) if prob.kind == "fit" else (float(prob.lp[0]), None)
        rec = {"workload": wl, "N": prob.N, "steps_per_window": steps}
        for S in (6, 7):
            ms = [r["ms"] for r in runs[S]]
            rec["S%d" % S] = {"ms": ms, "mean_ms": float(np.mean(ms)), "spread_ms": float(max(ms) - min(ms)),
                              "sm_mhz": [r["clocks"].get("sm_mhz") for r in runs[S]],
                              "reasons": [r["clocks"].get("reasons") for r in runs[S]]}
        rec["gain"] = 1.0 - rec["S6"]["mean_ms"] / rec["S7"]["mean_ms"]
        rec["gain_per_alternation"] = [1.0 - a["ms"] / b["ms"] for a, b in zip(runs[6], runs[7])]
        lp6, lp7 = out[6][0], out[7][0]
        rec["logpdf"] = {"S6": lp6, "S7": lp7, "rel_diff": abs(lp6 - lp7) / abs(lp7)}
        if out[6][1] is not None:
            a6, a7 = out[6][1], out[7][1]
            rec["alpha"] = {"max_rel_diff": float(np.max(np.abs(a6 - a7)) / np.max(np.abs(a7))),
                            "norm_rel_diff": float(np.linalg.norm(a6 - a7) / np.linalg.norm(a7))}
        if wl in ("C4", "C4h"):
            for S in (6, 7):
                eng.set_config(ozaki_slices=S, lookahead=0, profile_kernels=1)
                t, _, _ = bench.timed(prob, torch, flush, True, 3, 1)
                eng.set_config(lookahead=cfg0.lookahead, profile_kernels=cfg0.profile_kernels)
                rec["S%d" % S]["trailing_kernel_ms_per_step"] = t.get("trailing")
                eng.set_config(ozaki_slices=S)
                rec["S%d" % S]["parity_first_8192"] = bench.parity_check(wl, {"n": prob.N}, eng, torch, dev)
        eng.set_config(ozaki_slices=cfg0.ozaki_slices)
        print(json.dumps(rec), flush=True)
        del prob
        torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
