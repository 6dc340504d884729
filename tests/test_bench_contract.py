"""bench.py contract: the reference arm (CPU, no GPU needed) prints ONE JSON line with the keys the driver
reads, on the same metric / unit / config as our arm; under torchrun only rank 0 prints."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REQUIRED = {"impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
            "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"}


def _run(env_extra):
    env = dict(os.environ, LB2_BENCH_REF_ROWS="12000", **env_extra)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "0"], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    return [ln for ln in out.stdout.splitlines() if ln.strip()]


def test_reference_arm_prints_one_contract_line():
    lines = _run({})
    assert len(lines) == 1
    j = json.loads(lines[0])
    assert REQUIRED <= set(j)
    assert j["impl"] == "reference" and j["metric"] == "ivf_pq_index_build_mvec_per_s" and j["unit"] == "Mvec/s"
    assert j["higher_is_better"] is True and j["vs_baseline"] is None and j["value"] > 0
    assert j["cpu_baseline"]["kind"] == "port" and j["cpu_baseline"]["cores"] >= 1
    assert j["cpu_baseline"]["value"] == j["value"] and j["e2e"]["value"] == j["value"]
    assert j["e2e"]["h2d_bytes_per_step"] == 0 and j["e2e"]["d2h_bytes_per_step"] == 0
    assert "workload" in j["config"] and "model" not in j["config"]


def test_reference_arm_other_ranks_stay_silent():
    assert _run({"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"}) == []


def test_committed_bench_line_follows_the_contract():
    """profiles/bench_h100_C1.json is the line `python bench.py` printed on an H100 (profiles/README.md)."""
    j = json.load(open(os.path.join(ROOT, "profiles", "bench_h100_C1.json")))
    base = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
            "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"}
    assert base <= set(j)
    assert j["n_gpus"] == 1 and j["warmup"] >= 3 and j["higher_is_better"] is True and j["scaling"] == "weak"
    assert j["data"] == "synthetic" and j["dtype"] == "f32" and j["vs_baseline"] is None
    assert abs(j["value"] - 1e6 / (j["ms_per_step"] * 1e-3) / 1e6) < 1e-6 * j["value"]      # 1M rows per step
    r = j["roofline"]
    assert r["bound"] in ("hbm", "tensor") and r["unit"] in ("GB/s", "TFLOP/s")
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    # the dominant kernel's bytes follow bench.py's formula, and its rate follows from its measured launch time
    sys.path.insert(0, ROOT)
    import bench
    k = j["kernels"][r["kernel"]]
    assert r["algorithmic_bytes_per_launch"] == bench.KERNEL_BYTES[r["kernel"]](65536, 1_000_000)
    assert abs(r["avg_launch_ms"] - k["ms_per_step"] / k["launches_per_step"]) < 1e-9
    assert abs(r["achieved"] - r["algorithmic_bytes_per_launch"] / (r["avg_launch_ms"] * 1e-3) / 1e9) < 1e-6 * r["achieved"]
    assert r["kernel"] == max((f for f in j["kernels"] if f in bench.KERNEL_BYTES), key=lambda f: j["kernels"][f]["ms_per_step"])
    e = j["e2e"]
    assert e["h2d_bytes_per_step"] == 1_000_000 * 128 * 4 and e["d2h_bytes_per_step"] > 0 and 0 < e["value"] < j["value"]
    c = j["cpu_baseline"]
    assert c["kind"] in ("port", "reference") and c["cores"] >= 1 and c["value"] > 0 and c["sample"]
    assert j["gpu_launches"] > 0 and not set(j["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(j["clocks"])


def test_committed_round2_bench_lines_follow_the_contract():
    """profiles/bench_h100_C1.json (with the CPU baseline) and bench_h100_C1_no_cpu_baseline.json (run with
    --no-cpu-baseline) are lines `python bench.py` printed on an H100."""
    base = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
            "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline"}
    for name, with_cpu in (("bench_h100_C1.json", True), ("bench_h100_C1_no_cpu_baseline.json", False)):
        lines = [ln for ln in open(os.path.join(ROOT, "profiles", name)).read().splitlines() if ln.startswith("{")]
        j = json.loads(lines[-1])
        assert base <= set(j), name
        assert j["metric"] == "ivf_pq_index_build_mvec_per_s" and j["n_gpus"] == 1 and j["warmup"] >= 3
        assert abs(j["value"] - 1e6 / (j["ms_per_step"] * 1e-3) / 1e6) < 1e-6 * j["value"]
        r = j["roofline"]
        assert r["bound"] in ("hbm", "tensor") and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
        e = j["e2e"]
        assert e["h2d_bytes_per_step"] == 1_000_000 * 128 * 4 and e["d2h_bytes_per_step"] > 0 and 0 < e["value"] < j["value"]
        assert e["steps"] == j["steps"]                       # round 1 timed 3 e2e steps whatever --steps said
        assert j["gpu_launches"] > 0 and not set(j["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
        if with_cpu:
            c = j["cpu_baseline"]
            assert c["kind"] == "port" and c["cores"] >= 1 and c["value"] > 0 and "timed, not scaled" in c["sample"]
        q = j["query"]
        assert q["batch"] == 10000 and q["nprobes"] == 10 and 0 < q["recall_at_10"] <= 1
