"""bench.py output contract (CPU): the reference arm runs here end to end; the committed GPU bench line under
profiles/ carries every key a reader of bench.py's output relies on."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config", "e2e", "cpu_baseline"}


def _check_common(line):
    assert BASE_KEYS <= set(line), sorted(BASE_KEYS - set(line))
    assert line["metric"] == "images/sec" and line["unit"] == "images/sec" and line["higher_is_better"] is True
    assert line["scaling"] == "weak" and line["data"] == "synthetic" and "workload" in line["config"]
    assert line["value"] > 0 and line["ms_per_step"] > 0
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(line["e2e"])
    assert {"value", "unit", "cores", "kind", "sample"} <= set(line["cpu_baseline"])


def test_reference_arm_runs_on_cpu():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "1"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["steps"] == 1 and line["warmup"] == 1
    _check_common(line)
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
    # the unmodified reference when build() compiled it into oracle/_ref (git-ignored), else the port
    shipped = os.path.exists(os.path.join(ROOT, "oracle", "_ref", "main.pyc"))
    assert line["cpu_baseline"]["kind"] == ("reference" if shipped else "port")
    assert line["cpu_baseline"]["value"] == line["value"] and line["cpu_baseline"]["cores"] >= 1


def test_committed_gpu_bench_lines():
    for name, n in (("bench_h100_n1_b512.json", 1),):
        line = json.loads(open(os.path.join(ROOT, "profiles", name)).read().strip().splitlines()[-1])
        assert line["n_gpus"] == n and line["dtype"] == "bf16" and line["steps"] >= 1 and line["warmup"] >= 3
        _check_common(line)
        assert line["cpu_baseline"]["kind"] in ("reference", "port")
        assert line["gpu_launches"] > 0 and line["config"]["cuda_graphs"] is True
        assert line["host_enqueue_ms_per_step"] < 10.0          # the step is replayed from CUDA graphs
        assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(line["clocks"])
        assert not ({"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} & set(line["clocks"]["reasons"]))
        roof = line["roofline"]
        assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(roof)
        assert abs(roof["frac"] - roof["achieved"] / roof["peak"]) < 1e-9
        # e2e moves the step's inputs through pinned host memory: two fp32 views per image
        assert line["e2e"]["h2d_bytes_per_step"] >= 2 * 3 * 224 * 224 * 4 * 512 and line["e2e"]["d2h_bytes_per_step"] > 0
