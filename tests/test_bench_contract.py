"""bench.py contract (CPU part): the reference arm prints ONE JSON line with the required keys, and the
algorithmic-flop helper matches N^3/3 to leading order."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout + r.stderr
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["higher_is_better"] is False and d["unit"] == "ms" and d["vs_baseline"] is None
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert "workload" in d["config"] and "C4" in d["config"]["workload"]  # the same workload as the GPU arm at every N
    assert "extrapolated" in d["cpu_baseline"]["sample"]  # bounded N = 8192 sample, labelled


def test_trailing_flops_close_to_third_n_cubed():
    sys.path.insert(0, ROOT)
    import bench
    for n in (4096, 32768):
        assert abs(bench.trailing_flops(n) / (n ** 3 / 3.0) - 1.0) < 0.06
    assert abs(bench.trailing_flops(65536, 512) / (65536 ** 3 / 3.0) - 1.0) < 0.03


def test_reference_arm_other_workloads_are_bounded():
    """C2 runs in full; C3 / C5 samples are bounded and labelled"""
    sys.path.insert(0, ROOT)
    import bench
    cfg, scale, sample = bench.cpu_sample("C2", 4096)
    assert scale == 1.0 and cfg["X"].shape == (4096, 8)
    cfg, scale, sample = bench.cpu_sample("C5", 1000000)
    assert cfg["X"].shape[0] == 20000 and scale > 100 and "extrapolated" in sample
    cfg, scale, sample = bench.cpu_sample("C3", 16384)
    assert cfg["X"].shape[0] == 8192 and abs(scale - 8.0) < 1e-9 and cfg["Xs"].shape[0] == 5000
