"""tools/measure.py, the one place the benchmark tools record the card and time CUDA work (CPU only)."""
import ast
import glob
import importlib.util
import os
import runpy
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
TOOL_FILES = sorted(glob.glob(os.path.join(TOOLS, "*.py")))

_spec = importlib.util.spec_from_file_location("measure", os.path.join(TOOLS, "measure.py"))
measure = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(measure)


class _Props:
    uuid = "0e3e4a3c-1111-2222-3333-444455556666"


@pytest.fixture
def fake_device(monkeypatch):
    monkeypatch.setattr(torch.cuda, "get_device_properties", lambda i: _Props())
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda i: "Fake H100")


def test_card_asks_nvidia_smi_for_torch_device_0_by_uuid(fake_device, monkeypatch):
    calls = []

    def run(cmd, **kw):
        calls.append(cmd)
        return subprocess.CompletedProcess(cmd, 0, stdout="NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz\n", stderr="")

    monkeypatch.setattr(subprocess, "run", run)
    assert measure.card() == {"name": "Fake H100",
                              "name_power_limit_max_sm_clock": "NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz"}
    (cmd,) = calls
    assert cmd[0] == "nvidia-smi" and "--query-gpu=name,power.limit,clocks.max.sm" in cmd
    assert "-i" not in cmd and [a for a in cmd if a.startswith("--id")] == [f"--id=GPU-{_Props.uuid}"]


@pytest.mark.parametrize("outcome", ["missing", "timeout", "fails", "silent"])
def test_card_without_a_working_nvidia_smi_is_a_record(fake_device, monkeypatch, outcome):
    def run(cmd, **kw):
        if outcome == "missing":
            raise FileNotFoundError(2, "No such file or directory", "nvidia-smi")
        if outcome == "timeout":
            raise subprocess.TimeoutExpired(cmd, kw.get("timeout"))
        if outcome == "fails":
            return subprocess.CompletedProcess(cmd, 6, stdout="", stderr="No devices were found\n")
        return subprocess.CompletedProcess(cmd, 0, stdout="", stderr="")

    monkeypatch.setattr(subprocess, "run", run)
    rec = measure.card()
    assert rec["name"] == "Fake H100"
    smi = rec["name_power_limit_max_sm_clock"]
    if outcome == "silent":
        assert smi is None
    elif outcome == "fails":
        assert smi == "No devices were found"
    else:
        assert smi.startswith("unavailable: ")


def test_launch_ms_times_each_launch_in_order_and_takes_medians(monkeypatch):
    ran, ms = [], iter([5.0, 1.0, 3.0, 2.0, 4.0, 9.0])

    def event_ms(fn):
        fn()
        return next(ms)

    monkeypatch.setattr(measure, "event_ms", event_ms)
    got = measure.launch_ms({"a": lambda: ran.append("a"), "b": lambda: ran.append("b")}, 3)
    assert ran == ["a", "b"] * 3
    assert got == {"a": 4.0, "b": 2.0}


def _own_measurement(path):
    """Names of the CUDA-event constructions and nvidia-smi invocations in one tool's source."""
    found = []
    for node in ast.walk(ast.parse(open(path).read(), path)):
        if isinstance(node, ast.Attribute) and node.attr == "Event":
            found.append(f"line {node.lineno}: .Event")
        if isinstance(node, ast.ImportFrom) and any(a.name == "Event" for a in node.names):
            found.append(f"line {node.lineno}: import Event")
        if isinstance(node, ast.Constant) and isinstance(node.value, str) and node.value.split()[:1] == ["nvidia-smi"]:
            found.append(f"line {node.lineno}: {node.value!r}")
    return found


def test_only_measure_times_with_events_or_asks_nvidia_smi():
    assert _own_measurement(os.path.join(TOOLS, "measure.py"))          # the check sees what it looks for
    found = {os.path.basename(p): _own_measurement(p) for p in TOOL_FILES if os.path.basename(p) != "measure.py"}
    assert not {k: v for k, v in found.items() if v}, "use tools/measure.py instead of a copy"


PARSER_TOOLS = [os.path.basename(p) for p in TOOL_FILES if "ArgumentParser" in open(p).read()]


def test_parser_tools_are_found():
    assert {"bench_render.py", "bench_png.py", "bench_body_model.py", "bench_audio_frontend.py",
            "bench_lstm_pipeline.py", "bench_vq.py"} <= set(PARSER_TOOLS)


@pytest.mark.parametrize("tool", PARSER_TOOLS)
def test_tool_help_needs_no_gpu(tool, monkeypatch, capsys):
    # run as `python tools/<tool> --help` would: the script's directory first on sys.path
    monkeypatch.setattr(sys, "path", [TOOLS] + sys.path)
    monkeypatch.setattr(sys, "argv", [os.path.join(TOOLS, tool), "--help"])
    monkeypatch.setitem(sys.modules, "measure", measure)
    with pytest.raises(SystemExit) as exc:
        runpy.run_path(os.path.join(TOOLS, tool), run_name="__main__")
    assert exc.value.code == 0
    assert "usage:" in capsys.readouterr().out
