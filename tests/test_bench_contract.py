"""CPU: the parts of bench.py's contract that run without a GPU -- the `--impl reference` arm (the CPU oracle timed
through the same command line the driver uses) prints ONE JSON line with the agreed keys, and the result line of the GPU
arm committed under profiles/ (measured on an H100) carries the keys the measurement rules ask for."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    b = json.loads(lines[0])
    assert b["impl"] == "reference" and b["metric"] == "image_pairs_per_sec_256x192" and b["unit"] == "pairs/s"
    assert b["value"] > 0 and b["higher_is_better"] is True and b["n_gpus"] == 1
    assert b["cpu_baseline"]["kind"] == "port" and b["cpu_baseline"]["cores"] >= 1 and b["cpu_baseline"]["sample"]
    assert b["e2e"]["value"] == b["value"] and b["e2e"]["h2d_bytes_per_step"] == 0 and b["e2e"]["d2h_bytes_per_step"] == 0


def test_committed_gpu_line_has_the_contract_keys():
    path = os.path.join(ROOT, "profiles", "h100_bench.json")
    b = json.loads(open(path).readline())
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "gpu_launches", "clocks", "e2e", "roofline", "cpu_baseline"):
        assert k in b, k
    assert b["config"]["workload"].startswith("BASELINE.json configs[2]")
    assert b["gpu_launches"] > 0 and b["e2e"]["h2d_bytes_per_step"] > 0 and b["e2e"]["value"] <= b["value"] * 1.02
    r = b["roofline"]
    assert r["bound"] == "tensor" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-6 and "traffic" in r   # DRAM traffic: not measured
    assert b["check"]["l1_rel_depth0_vs_cpu_oracle_fp32"] < 1e-4 and b["check"]["tc_timeouts"] == 0
    assert b["device"]["name"].startswith("NVIDIA H100") and b["device"]["power_limit_w"] > 0   # what the line was measured on
