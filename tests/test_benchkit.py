"""tools/benchkit.py, the plumbing the benchmark scripts share, and the scripts' imports, without a GPU."""
import glob
import importlib.util
import json
import os
import stat
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
# run_ops_once launches its ops at import: it has no main
SCRIPTS = sorted(p for p in glob.glob(os.path.join(TOOLS, "*.py")) if os.path.basename(p) != "run_ops_once.py")


def load(path):
    spec = importlib.util.spec_from_file_location("tools_" + os.path.basename(path)[:-3], path)
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    return module


@pytest.fixture
def benchkit(monkeypatch):
    monkeypatch.syspath_prepend(TOOLS)   # as when a script runs as python tools/<name>.py
    return load(os.path.join(TOOLS, "benchkit.py"))


@pytest.fixture
def device(monkeypatch):
    """torch on card 1 of several, a named H100 with a fixed UUID."""
    props = {1: types.SimpleNamespace(name="NVIDIA H100 80GB HBM3", uuid="6f0c1e2a-3b4d-5e6f-7081-92a3b4c5d6e7")}
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 1)
    monkeypatch.setattr(torch.cuda, "get_device_properties", lambda i: props[i])


def fake_nvidia_smi(monkeypatch, tmp_path, script):
    exe = tmp_path / "nvidia-smi"
    exe.write_text("#!/bin/sh\n" + script)
    exe.chmod(exe.stat().st_mode | stat.S_IXUSR)
    monkeypatch.setenv("PATH", str(tmp_path))


def test_device_info_queries_the_timed_card(benchkit, device, monkeypatch, tmp_path):
    fake_nvidia_smi(monkeypatch, tmp_path, 'echo "$@" > "%s/args"\necho "400.00 W, 1980 MHz"\n' % tmp_path)
    assert benchkit.device_info() == {"gpu": "NVIDIA H100 80GB HBM3", "power_limit": "400.00 W", "max_sm_clock": "1980 MHz"}
    args = (tmp_path / "args").read_text().split()
    assert args[args.index("-i") + 1] == "GPU-6f0c1e2a-3b4d-5e6f-7081-92a3b4c5d6e7"


def test_device_info_without_nvidia_smi(benchkit, device, monkeypatch, tmp_path):
    monkeypatch.setenv("PATH", str(tmp_path))
    assert benchkit.device_info() == {"gpu": "NVIDIA H100 80GB HBM3", "power_limit": "unknown (FileNotFoundError)",
                                      "max_sm_clock": "unknown (FileNotFoundError)"}


def test_rows_carry_the_card_and_append(benchkit, device, monkeypatch, tmp_path, capsys):
    fake_nvidia_smi(monkeypatch, tmp_path, 'echo "700.00 W, 1980 MHz"\n')
    out = tmp_path / "runs" / "rows.jsonl"
    rows = benchkit.Rows(str(out))
    rows.add({"bench": "a", "ms": 1.5})
    rows.add({"bench": "b", "ms": 2.5})
    card = {"gpu": "NVIDIA H100 80GB HBM3", "power_limit": "700.00 W", "max_sm_clock": "1980 MHz"}
    expected = [dict({"bench": "a", "ms": 1.5}, **card), dict({"bench": "b", "ms": 2.5}, **card)]
    assert [json.loads(ln) for ln in capsys.readouterr().out.splitlines()] == expected
    assert not out.exists()   # nothing is written before the run is through
    rows.save()
    rows.save()
    assert [json.loads(ln) for ln in out.read_text().splitlines()] == expected * 2
    benchkit.Rows(None).save()   # no --out: print only


def test_summary(benchkit):
    assert benchkit.summary([3.0, 1.0, 10.0, 2.0]) == {"ms": 2.5, "ms_min": 1.0, "ms_max": 10.0, "steps": 4}
    assert benchkit.summary([4.0, 0.5, 2.0]) == {"ms": 2.0, "ms_min": 0.5, "ms_max": 4.0, "steps": 3}


@pytest.mark.parametrize("path", SCRIPTS, ids=os.path.basename)
def test_script_imports(path, benchkit, monkeypatch):
    for v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):   # bench_datareader sets them at import
        monkeypatch.setenv(v, "1")
    module = load(path)
    if os.path.basename(path) != "benchkit.py":
        assert callable(module.main)
