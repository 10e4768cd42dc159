"""bench.py contract (CPU part): the reference arm prints ONE JSON line with the keys a caller
reads, and the cost-model extrapolation is self-consistent.  (The GPU arm's JSON line from an
H100 run is committed under profiles/.)"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json(monkeypatch, capsys):
    import bench
    real = bench.run_cpu_sample
    monkeypatch.setattr(bench, "run_cpu_sample", lambda n_s=None, reps=1: real(512, reps))
    args = type("A", (), dict(gpus=1, steps=2, warmup=1))()
    bench.reference_main(args)
    line = capsys.readouterr().out.strip().splitlines()[-1]
    d = json.loads(line)
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e", "gpu_launches"):
        assert k in d, k
    assert d["impl"] == "reference" and d["unit"] == "points/s" and d["dtype"] == "f64" and d["vs_baseline"] is None
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert "workload" in d["config"]


def test_non_zero_ranks_of_reference_arm_exit_quietly():
    env = dict(os.environ, RANK="3", WORLD_SIZE="8", LOCAL_RANK="3")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "8"],
                       capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_extrapolation_model():
    import bench
    t = dict(assemble=1.0, chol=2.0, solve=0.5, posterior=3.0)
    # doubling N: assemble x4, chol x8, solves x4, posterior x4 (x N*/N* ratio)
    assert np.isclose(bench.cpu_extrapolate(t, 100, 10, 200, 10), 4 + 16 + 2 + 12)
    assert np.isclose(bench.cpu_extrapolate(t, 100, 10, 100, 20), 1 + 2 + 0.5 + 6)


def test_committed_gpu_bench_line_has_contract_keys():
    d = json.loads(open(os.path.join(ROOT, "profiles", "bench_h100_1gpu.json")).read().strip().splitlines()[-1])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "cpu_baseline", "clocks"):
        assert k in d, k
    assert d["roofline"]["bound"] == "tensor" and 0 < d["roofline"]["frac"] <= 1.05
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["gpu_launches"] > 0 and d["warmup"] >= 3
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
