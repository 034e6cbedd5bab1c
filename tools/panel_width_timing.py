"""Alternate arms of `bench.py --quick` in one session on one card; an arm is a tree (built, its libagp.so in place) plus
environment settings, so it compares outer panel widths (AGP_NB) in one tree, or this tree against a build of another
revision:
  - the card's name, power limit and maximum SM clock, first and last;
  - per workload, `reps` alternations of every arm (C4: 5 steps, C4h: 10, C2: 20, C3: 10): device time per step, with
    the SM clock and clock-event reasons nvidia-smi saw during each run, and the outputs (`--dump-outputs`) compared bit
    for bit with the first arm's, or their largest relative difference where they differ;
  - with --trailing, one run per arm with look-ahead off and the kernels timed (AGP_LOOKAHEAD=0 AGP_PROFILE=1): the
    trailing updates' summed launch time per step, as bench.py's roofline pass takes it;
  - with --bench-line, one full `bench.py` line of the first arm.
Prints one JSON object per measurement.
Usage: python tools/panel_width_timing.py --arm nb512=.:AGP_NB=512 --arm nb1024=.:AGP_NB=1024 [--reps 3]
       [--workloads C4,C4h] [--trailing] [--bench-line] [--out DIR]
(an arm is NAME=TREE[:VAR=VALUE[,VAR=VALUE...]]; TREE is relative to the repository root)"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = {"C4": 5, "C4h": 10, "C2": 20, "C3": 10}


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return {"query": q, "value": r.stdout.strip()}


def parse_arm(s):
    name, rest = s.split("=", 1)
    tree, _, envs = rest.partition(":")
    env = dict(kv.split("=", 1) for kv in envs.split(",") if kv)
    return name, os.path.abspath(os.path.join(ROOT, tree)), env


def bench(tree, args, env=None):
    """one bench.py process of `tree`; returns its JSON line and what nvidia-smi saw while it ran (samples with the GPU
    busy: utilisation >= 50 %)"""
    q = "clocks.sm,utilization.gpu,power.draw,clocks_event_reasons.active"
    smi = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-lms", "200"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    try:
        r = subprocess.run([sys.executable, os.path.join(tree, "bench.py")] + args, cwd=tree, capture_output=True, text=True,
                           env=dict(os.environ, **(env or {})))
    finally:
        smi.terminate()
        smi_out, _ = smi.communicate()
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError("bench.py %s in %s failed:\n%s\n%s" % (" ".join(args), tree, r.stdout[-2000:], r.stderr[-4000:]))
    busy = []
    for l in smi_out.splitlines():
        f = [x.strip() for x in l.split(",")]
        try:
            if len(f) == 4 and float(f[1]) >= 50:
                busy.append((float(f[0]), float(f[2]), f[3]))
        except ValueError:
            pass
    clocks = {"samples": len(busy)}
    if busy:
        mhz = [b[0] for b in busy]
        clocks.update(sm_mhz_median=float(np.median(mhz)), sm_mhz_min=min(mhz), sm_mhz_max=max(mhz),
                      power_w_median=float(np.median([b[1] for b in busy])), reasons=sorted({b[2] for b in busy}))
    return json.loads(lines[-1]), clocks


def compare_outputs(d0, d1):
    """per output: "identical", or the largest difference relative to the first arm's largest magnitude"""
    out = {}
    for name in sorted(os.listdir(d0)):
        a, b = np.load(os.path.join(d0, name)), np.load(os.path.join(d1, name))
        if a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes():
            out[name[:-4]] = "identical"
        else:
            a64, b64 = a.astype(np.float64), b.astype(np.float64)
            out[name[:-4]] = float(np.max(np.abs(a64 - b64)) / max(np.max(np.abs(a64)), 1e-300))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", action="append", required=True, help="NAME=TREE[:VAR=VALUE,...]")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default="C4,C4h")
    ap.add_argument("--trailing", action="store_true")
    ap.add_argument("--bench-line", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the dumped outputs (default: a temporary one)")
    a = ap.parse_args()
    arms = [parse_arm(s) for s in a.arm]
    out = a.out or tempfile.mkdtemp(prefix="panel_width_")
    print(json.dumps({"card": card(), "arms": {n: {"tree": t, "env": e} for n, t, e in arms}}), flush=True)
    for wl in a.workloads.split(","):
        steps = STEPS[wl]
        runs = {n: [] for n, _, _ in arms}
        for rep in range(a.reps):
            for n, tree, env in (arms if rep % 2 == 0 else arms[::-1]):
                d = os.path.join(out, wl, n, str(rep))
                line, clocks = bench(tree, ["--workload", wl, "--quick", "--steps", str(steps), "--dump-outputs", d], env)
                runs[n].append({"ms": line["value"], "cholesky_ms": line["phases_ms"].get("cholesky"), "clocks": clocks,
                                "result": line.get("result"), "dump": d})
        rec = {"workload": wl, "steps_per_run": steps}
        first = arms[0][0]
        for n, _, _ in arms:
            ms = [r["ms"] for r in runs[n]]
            rec[n] = {"ms": ms, "mean_ms": float(np.mean(ms)), "spread_ms": float(max(ms) - min(ms)),
                      "cholesky_ms": [r["cholesky_ms"] for r in runs[n]], "result": [r["result"] for r in runs[n]],
                      "clocks": [r["clocks"] for r in runs[n]]}
            if n != first:
                rec[n]["change_vs_" + first] = rec[n]["mean_ms"] / rec[first]["mean_ms"] - 1.0
                rec[n]["change_per_alternation"] = [r["ms"] / f["ms"] - 1.0 for r, f in zip(runs[n], runs[first])]
                rec[n]["outputs_vs_" + first] = [compare_outputs(f["dump"], r["dump"]) for r, f in zip(runs[n], runs[first])]
        print(json.dumps(rec), flush=True)
    if a.trailing:
        for n, tree, env in arms:
            line, clocks = bench(tree, ["--workload", "C4", "--quick", "--steps", "3", "--warmup", "1"],
                                 dict(env, AGP_LOOKAHEAD="0", AGP_PROFILE="1"))
            print(json.dumps({"workload": "C4", "arm": n, "lookahead": 0, "step_ms": line["value"],
                              "trailing_ms_per_step": line["phases_ms"].get("trailing"), "clocks": clocks}), flush=True)
    if a.bench_line:
        n, tree, env = arms[0]
        line, clocks = bench(tree, ["--gpus", "1", "--steps", "5", "--warmup", "3", "--no-c2"], env)
        print(json.dumps({"arm": n, "bench_line": line, "clocks_seen": clocks}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
