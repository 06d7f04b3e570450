"""The bench lines committed under profiles/ (measured on one H100 by `bench.py`) carry every key of the bench contract —
a schema check of the evidence files, so that a refactor of bench.py that drops a key is caught in the CPU suite."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
        "dtype", "data", "config", "e2e", "gpu_launches", "clocks")


def _line(name):
    with open(os.path.join(ROOT, "profiles", name)) as f:
        return json.loads(f.read().strip().splitlines()[-1])


def test_headline_line_has_the_whole_contract():
    d = _line("h100_bench_line.json")
    for k in BASE + ("roofline", "cpu_baseline"):
        assert k in d, k
    assert d["metric"] == "speech_tokens_per_s" and d["unit"] == "tokens/s" and d["higher_is_better"] is True
    assert d["n_gpus"] == 1 and d["warmup"] >= 3 and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert "workload" in d["config"] and "model" not in d["config"]
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in r, k
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    if r["traffic"] is not None:                                                # only with a committed ncu capture
        assert 0.9 < r["traffic"] / r["algorithmic_bytes_per_step"] < 1.1      # no wasted re-reads of the weight stream
    c = d["cpu_baseline"]
    for k in ("value", "unit", "cores", "kind", "sample"):
        assert k in c, k
    assert c["kind"] == "port" and c["cores"] >= 1
    e = d["e2e"]
    assert e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and e["unit"] == d["unit"]
    assert e["value"] <= d["value"] * 1.001                                     # host copies inside the timed region
    assert d["gpu_launches"] > 0
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert abs(d["value"] - d["n_gpus"] * d["steps"] * 256 / (d["ms_per_step"] * d["steps"] / 1000.0)) / d["value"] < 1e-6


@pytest.mark.parametrize("name,ngpu", [("h100_bench_config3_n1.json", 1), ("h100_bench_config5_n1.json", 1)])
def test_job_lines(name, ngpu):
    d = _line(name)
    for k in BASE:
        assert k in d, k
    assert d["n_gpus"] == ngpu and d["scaling"] == "strong"
    pr = d["per_rank"]
    assert len(pr["busy_s"]) == ngpu and sum(pr["tokens"]) == d["config"]["speech_tokens"]
    # whole-job throughput = all tokens / the slowest rank's wall time
    assert abs(d["value"] - d["config"]["speech_tokens"] / (d["ms_per_step"] / 1000.0)) / d["value"] < 1e-6
    assert max(pr["busy_s"]) <= d["ms_per_step"] / 1000.0 + 1e-6
