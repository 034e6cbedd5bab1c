"""This tree against a baseline tree (another revision with its own built libagp.so), each run through its own bench.py in
a fresh process, alternated in one session on one card:
  - the card's name, power limit and maximum SM clock, first and last;
  - C4 (`reps` alternations of 5 steps) and C4h (`reps` of 10), `bench.py --quick`: device time per step, with the SM
    clock and clock-event reasons nvidia-smi saw during each run;
  - C2 and C3 (two alternations each), which do not run the eight-bit kernel, as a control;
  - the outputs of every run (`--dump-outputs`: logpdf and alpha; mean and var for C3) compared bit for bit between the
    trees;
  - one C4 run of this tree with bounded CTAs of twice as many tiles (AGP_OZAKI_CHUNK=32);
  - one full `bench.py` line of this tree (trailing-kernel ms per step and its share of the int8 peak).
Prints one JSON object per measurement.
Usage: python tools/ozaki8_tile_timing.py BASELINE_TREE [--reps 3] [--out DIR] [--workloads C4,C4h,C2,C3] [--no-bench-line]
(--workloads and --no-bench-line split the session where one process may not run for the ten-odd minutes it takes)"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return {"query": q, "value": r.stdout.strip()}


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


def same_outputs(d0, d1):
    out = {}
    for name in sorted(os.listdir(d0)):
        a, b = np.load(os.path.join(d0, name)), np.load(os.path.join(d1, name))
        out[name[:-4]] = bool(a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("baseline", help="another revision's tree, built (its libagp.so in place)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the dumped outputs (default: a temporary one)")
    ap.add_argument("--workloads", default="C4,C4h,C2,C3")
    ap.add_argument("--no-bench-line", action="store_true")
    a = ap.parse_args()
    trees = {"new": ROOT, "base": os.path.abspath(a.baseline)}
    out = a.out or tempfile.mkdtemp(prefix="ozaki8_tile_")
    print(json.dumps({"card": card()}), flush=True)
    todo = a.workloads.split(",")
    for wl, steps, reps in (("C4", 5, a.reps), ("C4h", 10, a.reps), ("C2", 20, 2), ("C3", 10, 2)):
        if wl not in todo:
            continue
        runs = {k: [] for k in trees}
        for rep in range(reps):
            for k in (("new", "base") if rep % 2 == 0 else ("base", "new")):
                d = os.path.join(out, wl, k, str(rep))
                line, clocks = bench(trees[k], ["--workload", wl, "--quick", "--steps", str(steps), "--dump-outputs", d])
                runs[k].append({"ms": line["value"], "cholesky_ms": line["phases_ms"].get("cholesky"), "clocks": clocks,
                                "dump": d})
        rec = {"workload": wl, "steps_per_run": steps}
        for k in trees:
            ms = [r["ms"] for r in runs[k]]
            rec[k] = {"ms": ms, "mean_ms": float(np.mean(ms)), "spread_ms": float(max(ms) - min(ms)),
                      "cholesky_ms": [r["cholesky_ms"] for r in runs[k]], "clocks": [r["clocks"] for r in runs[k]]}
        rec["gain"] = 1.0 - rec["new"]["mean_ms"] / rec["base"]["mean_ms"]
        rec["gain_per_alternation"] = [1.0 - n["ms"] / b["ms"] for n, b in zip(runs["new"], runs["base"])]
        rec["outputs_identical"] = [same_outputs(n["dump"], b["dump"]) for n, b in zip(runs["new"], runs["base"])]
        print(json.dumps(rec), flush=True)
    if "C4" in todo:
        line, clocks = bench(ROOT, ["--workload", "C4", "--quick", "--steps", "5"], env={"AGP_OZAKI_CHUNK": "32"})
        print(json.dumps({"workload": "C4", "tree": "new", "AGP_OZAKI_CHUNK": 32, "ms": line["value"], "clocks": clocks}),
              flush=True)
    if not a.no_bench_line:
        line, clocks = bench(ROOT, ["--gpus", "1", "--steps", "5", "--warmup", "3", "--no-c2"])
        print(json.dumps({"bench_line": line, "clocks_seen": clocks}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
