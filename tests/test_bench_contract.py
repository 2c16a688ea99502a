"""The committed bench lines (profiles/) carry every key of the bench.py output format -- a guard against drifting away
from what consumers of the line parse.  CPU only: it reads the JSON written by the last GPU run."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _last_json_line(path):
    with open(path) as fh:
        lines = [ln for ln in fh.read().splitlines() if ln.startswith("{")]
    return json.loads(lines[-1])


def test_committed_bench_line_has_the_contract_keys():
    d = _last_json_line(os.path.join(ROOT, "profiles", "h100_bench.json"))
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "cpu_baseline", "clocks"):
        assert key in d, key
    assert d["higher_is_better"] is True and d["scaling"] == "weak" and d["warmup"] >= 3 and d["gpu_launches"] > 0
    assert "workload" in d["config"] and "model" not in d["config"]
    for key in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert key in d["e2e"], key
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
    for key in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert key in d["roofline"], key
    assert d["roofline"]["frac"] == pytest.approx(d["roofline"]["achieved"] / d["roofline"]["peak"])
    for key in ("value", "unit", "cores", "kind", "sample"):
        assert key in d["cpu_baseline"], key
    for key in ("sm_mhz", "sm_max_mhz", "reasons"):
        assert key in d["clocks"], key
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    # configs 3, 5 and 1 and the --quantize configuration ride on the same line
    cfg = d["configs"]
    for key in ("value", "unit", "ms_per_step", "e2e", "roofline", "stage_ms_per_step", "gpu_launches"):
        assert key in cfg["config3_sup"], key
    assert len(cfg["config5_sup_sweep"]) == 3 and all(b["value"] > 0 for b in cfg["config5_sup_sweep"])
    assert cfg["config1_fast_cpu"]["value"] > 0 and cfg["hac_quantize_int8"]["value"] > 0


def test_committed_reference_arm_line():
    d = _last_json_line(os.path.join(ROOT, "profiles", "h100_bench_reference.json"))
    assert d["impl"] == "reference" and d["cpu_baseline"]["kind"] in ("port", "reference")
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["e2e"]["value"] == d["value"] and d["unit"] == "samples/s"
