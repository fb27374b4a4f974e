"""The bench line committed under profiles/ (bench_r02_default.json: one H100, the default S8 workload) carries every key
bench.py's output names (roofline, cpu_baseline, e2e, clocks, gpu_launches), with consistent values.  Guards the format against drift: bench.py itself
needs a GPU, its committed output does not."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
        "data", "config", "e2e", "gpu_launches", "clocks", "roofline"]


def _line(name):
    text = open(os.path.join(ROOT, "profiles", name)).read().strip().splitlines()
    return json.loads([t for t in text if t.startswith("{")][-1])


@pytest.mark.parametrize("name,n", [("bench_r02_default.json", 1)])
def test_committed_bench_lines_follow_the_contract(name, n):
    d = _line(name)
    for k in BASE:
        assert k in d, k
    assert d["n_gpus"] == n and d["unit"] == "queries/s" and d["higher_is_better"] is True and d["data"] == "synthetic"
    assert d["warmup"] >= 3 and d["steps"] >= 1
    assert "workload" in d["config"] and not any(k in d["config"] for k in ("model", "seq_len", "global_batch"))
    batch = d["config"]["batch"]
    assert abs(d["value"] - batch * 1e3 / d["ms_per_step"]) < 1e-6 * d["value"]          # value = queries per step / step time
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in r, k
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    e = d["e2e"]
    assert e["unit"] == d["unit"] and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and e["value"] != d["value"]
    c = d["clocks"]
    assert not any(x in c["reasons"] for x in ("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"))
    assert c["sm_mhz"] > 0 and c["sm_mhz"] >= 0.9 * c["sm_max_mhz"]
    assert d["gpu_launches"] > 0
    cpu = d["cpu_baseline"]
    for k in ("value", "unit", "cores", "kind", "sample"):
        assert k in cpu, k
    assert cpu["kind"] in ("port", "reference") and cpu["unit"] == d["unit"]
    assert d["scaling"] == "weak" and d["vs_baseline"] is None
