"""CPU test: the committed bench lines (profiles/bench_h100*.json, produced by `python bench.py` on an H100) carry every key the
bench contract names, with consistent values -- a regression net for bench.py's output format."""
import json
import os

import pytest

from conftest import ROOT


def load(name):
    p = os.path.join(ROOT, "profiles", name)
    if not os.path.exists(p):
        pytest.skip(name + " not committed")
    return json.load(open(p))


def check_common(d, cpu_baseline=True):
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
              "config", "e2e", "cpu_baseline"):
        assert k in d, k
    assert d["unit"] == "frames/s" and d["higher_is_better"] is True and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert "workload" in d["config"] and "model" not in d["config"]
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"])
    if cpu_baseline:   # (bench.py --no-cpu-baseline leaves it null)
        assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"]) and d["cpu_baseline"]["kind"] in ("reference", "port")


def test_h100_line():
    d = load("bench_h100.json")
    check_common(d)
    assert d["output_check"] == "matches the stored checksum"                         # the step's integer outputs, hashed inside the run
    assert d["config"]["workload"].startswith("c2_720p") and d["config"]["batch_frames_per_step"] == 64
    assert d["n_gpus"] == 1 and d["warmup"] >= 3 and d["gpu_launches"] > 0 and d["data"] == "synthetic"
    assert abs(d["value"] - 64 * 1e3 / d["ms_per_step"]) < 1e-6 * d["value"]          # 64 frames per step
    assert d["e2e"]["h2d_bytes_per_step"] == 64 * 1280 * 720 * 4 and d["e2e"]["d2h_bytes_per_step"] > 0
    assert d["e2e"]["value"] < d["value"]                                             # copies inside the timed region
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert abs(r["achieved"] - r["algorithmic_bytes_per_launch"] / (r["launch_ms"] * 1e-3) / 1e9) < 1e-6 * r["achieved"]
    c = d["clocks"]
    assert c["sm_mhz"] >= 0.9 * c["sm_max_mhz"] and not set(c["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    sysapi = d["stats"]["tracking_stages_us"]["system_api"]
    assert sysapi["status_counts"]["1"] > 20 and sysapi["concurrent_streams"]["all_streams_bit_identical"] is True


def test_reference_line():
    d = load("bench_h100_reference.json")
    check_common(d)
    assert d["impl"] == "reference" and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"] == d["cpu_baseline"]["value"]
    assert d["config"] == load("bench_h100.json")["config"]                            # same config dict as the repo arm


def test_c3_line():
    d = load("bench_h100_c3.json")
    check_common(d, cpu_baseline=False)
    assert d["config"]["frame"] == "1920x1080 RGBA" and d["config"]["features_per_frame"] == 2000
    assert abs(d["value"] - d["config"]["batch_frames_per_step"] * 1e3 / d["ms_per_step"]) < 1e-6 * d["value"]
    assert d["roofline"]["frac"] > 0.2
