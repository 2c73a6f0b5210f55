"""The committed bench lines under profiles/ carry every key of the bench.py contract (a format regression would make the
driver's BENCH_rNN.json unreadable); and bench.py's argument defaults stay inside the contract (N = 1, W >= 3)."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
        "dtype", "data", "config", "e2e"]


def _line(name):
    with open(os.path.join(ROOT, "profiles", name)) as f:
        return json.loads([l for l in f if l.startswith("{")][-1])


@pytest.mark.parametrize("name", ["bench_h100.json", "bench_h100_per_op.json", "bench_h100_13b.json", "bench_h100_13b_act.json",
                                  "bench_h100_33b_g32_act.json", "bench_h100_65b_seq4096.json"])
def test_bench_line_keys(name):
    if not os.path.exists(os.path.join(ROOT, "profiles", name)):
        pytest.skip(name + " not committed yet")
    d = _line(name)
    for k in BASE + ["gpu_launches", "clocks", "roofline"]:
        assert k in d, k
    assert "workload" in d["config"] and "model" not in d["config"]
    assert set(d["e2e"]) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} and d["e2e"]["h2d_bytes_per_step"] > 0
    assert d["clocks"] is None or set(d["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}
    r = d["roofline"]
    assert set(r) >= {"bound", "achieved", "peak", "unit", "frac", "traffic"} and r["bound"] in ("hbm", "tensor")
    assert r["frac"] is None or abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-3
    assert d["gpu_launches"] > 0 and d["warmup"] >= 3 and d["higher_is_better"] is True
    if d["n_gpus"] == 1:
        c = d["cpu_baseline"]
        assert c is not None and set(c) >= {"value", "unit", "cores", "kind", "sample"} and c["kind"] in ("reference", "port")
        assert abs(d["value"] - 1000.0 / d["ms_per_step"]) < 0.5


def test_reference_line_keys():
    d = _line("bench_h100_reference.json")
    for k in BASE + ["impl", "cpu_baseline"]:
        assert k in d, k
    assert d["impl"] == "reference" and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]


def test_bench_defaults():
    import importlib.util
    import sys
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    argv, sys.argv = sys.argv, ["bench.py"]
    try:
        a = m.parse()
    finally:
        sys.argv = argv
    assert a.gpus == 1 and a.warmup >= 3 and a.steps >= 8 and a.impl != "reference"


def test_profiles_index_names_existing_files():
    import re
    idx = open(os.path.join(ROOT, "profiles", "README.md")).read()
    names = re.findall(r"`([A-Za-z0-9_]+\.(?:json|jsonl|csv|txt))`", idx)
    assert names
    for name in names:
        assert os.path.exists(os.path.join(ROOT, "profiles", name)), name
