"""bench.py contract that can be checked without a GPU: the reference arm (the unmodified reference
from oracle/_ref when __graft_entry__.build() installed it, else the CPU port of its generation,
oracle/reference_port.py) prints exactly ONE JSON line on stdout with
the keys the driver reads; our own arm refuses to run without the CUDA library / a GPU."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench(*args, timeout=300):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True,
                          timeout=timeout, cwd=ROOT)


def test_reference_arm_prints_one_json_line():
    r = _bench("--impl", "reference", "--workload", "cartpole", "--steps", "1", "--warmup", "0")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "generations/s" and d["higher_is_better"] is True
    assert d["n_gpus"] == 1 and d["steps"] == 1 and d["value"] > 0 and d["ms_per_step"] > 0
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["value"] == d["value"] and "population_size=" in cb["sample"]
    assert d["config"]["workload"].startswith("cartpole") and d["config"]["population_size"] == 4096


def test_our_arm_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    r = _bench("--steps", "1", "--no-cpu-baseline")
    assert r.returncode != 0 and r.stdout.strip() == ""          # no JSON line, no silent CPU fallback
