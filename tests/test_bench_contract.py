"""CPU: the bench.py contract.  (a) `--impl reference` runs here (it is the host-core arm) and prints
one JSON line with the agreed keys; (b) the committed GPU snapshots under profiles/ (one H100) carry
every key of the contract."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config", "e2e"}


def test_reference_arm_prints_one_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and BASE_KEYS <= set(d)
    assert d["metric"] == "images/sec (480x640, K=9) backbone+vote" and d["unit"] == "images/sec"
    assert d["value"] > 0 and d["e2e"]["value"] == d["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["value"] == d["value"]
    assert "workload" in d["config"] and "model" not in d["config"]


def test_round2_snapshot_has_the_new_blocks():
    """profiles/bench_n1_h100.json: uint8 end-to-end input, vote roofline, config 4 measured in the same line."""
    d = json.load(open(os.path.join(ROOT, "profiles", "bench_n1_h100.json")))
    assert BASE_KEYS | {"gpu_launches", "clocks", "roofline", "roofline_vote", "config4", "cpu_baseline"} <= set(d)
    assert d["e2e"]["h2d_bytes_per_step"] == 16 * 480 * 640 * 3                   # raw uint8 HWC images
    rv = d["roofline_vote"]
    assert {"layer_ms", "tests", "tests_per_s", "alg_hbm_gbs", "alg_hbm_frac"} <= set(rv)
    c4 = d["config4"]
    assert {"value", "e2e", "roofline_vote", "workload"} <= set(c4) and "with_mean" in c4["workload"]
    assert c4["e2e"]["d2h_bytes_per_step"] == 16 * 9 * 2 * 4 * 3                   # keypoints + covariances


def test_committed_gpu_snapshot_has_the_contract_keys():
    d = json.load(open(os.path.join(ROOT, "profiles", "bench_n1_f32_h100.json")))
    assert BASE_KEYS | {"gpu_launches", "clocks", "roofline", "cpu_baseline"} <= set(d)
    assert d["n_gpus"] == 1 and d["warmup"] >= 3 and d["gpu_launches"] > 0
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"])
    assert d["e2e"]["h2d_bytes_per_step"] == 16 * 3 * 480 * 640 * 4
    r = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac"} <= set(r)
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-3 and r["bound"] in ("hbm", "tensor")
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(d["clocks"])
    assert not {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} & set(d["clocks"]["reasons"])
    assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"])
    assert "workload" in d["config"] and "model" not in d["config"]
