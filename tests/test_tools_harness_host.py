"""CPU: the benchmark tools' shared harness (tools/_harness.py).  Every tools/bench_*.py imports without running
anything, so every helper it takes from the harness or another tool resolves; card() asks nvidia-smi for the card by
UUID and never raises; every timer refuses to run without CUDA."""
import glob
import importlib
import os
import subprocess
import sys
import types

import pytest
import torch

from conftest import ROOT

TOOLS = os.path.join(ROOT, "tools")
BENCHES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(TOOLS, "bench_*.py")))
UUID = "4a6b1c2d-0e1f-2a3b-4c5d-6e7f8a9b0c1d"


@pytest.fixture
def harness(monkeypatch):
    monkeypatch.syspath_prepend(TOOLS)
    return importlib.import_module("_harness")


@pytest.fixture
def smi(harness, monkeypatch):
    """Fakes the device properties; returns the list of nvidia-smi calls, answered by `smi.answer`."""
    calls = []
    ns = types.SimpleNamespace(calls=calls, answer=None)

    def props(dev):
        calls.append(("props", dev))
        return types.SimpleNamespace(name="NVIDIA H100 80GB HBM3", uuid=UUID)

    def run(cmd, **kw):
        calls.append((cmd, kw))
        if isinstance(ns.answer, BaseException):
            raise ns.answer
        return subprocess.CompletedProcess(cmd, 0, stdout=ns.answer, stderr="")
    monkeypatch.setattr(harness.torch.cuda, "get_device_properties", props)
    monkeypatch.setattr(harness.torch.cuda, "current_device", lambda: 2)
    monkeypatch.setattr(harness.subprocess, "run", run)
    return ns


@pytest.mark.parametrize("name", BENCHES)
def test_every_tool_imports_without_running(name, harness, monkeypatch, capsys):
    monkeypatch.setattr(sys, "path", list(sys.path))       # the tools' own path inserts do not outlive the test
    monkeypatch.setattr(subprocess, "run", lambda *a, **k: pytest.fail(f"{name} ran a process at import"))
    mod = importlib.import_module(name)
    assert callable(mod.main)
    assert capsys.readouterr().out == ""


def test_card_queries_the_measured_device_by_uuid(harness, smi):
    smi.answer = "NVIDIA H100 80GB HBM3, 700.00 W, 1755 MHz, 1980 MHz\n"
    assert harness.card() == {"name": "NVIDIA H100 80GB HBM3", "power_limit": "700.00 W", "sm_clock": "1755 MHz",
                              "max_sm_clock": "1980 MHz"}
    (_, dev), (cmd, kw) = smi.calls
    assert dev == 2                                         # the current device
    assert cmd[0] == "nvidia-smi" and f"--id=GPU-{UUID}" in cmd
    assert "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm" in cmd and "--format=csv,noheader" in cmd
    assert kw["timeout"] > 0
    harness.card(torch.device("cuda", 5))
    assert smi.calls[2] == ("props", torch.device("cuda", 5))


@pytest.mark.parametrize("answer", [subprocess.TimeoutExpired("nvidia-smi", 30), FileNotFoundError("nvidia-smi"),
                                    subprocess.CalledProcessError(6, "nvidia-smi"), "No devices were found\n", ""])
def test_card_reports_a_failed_query_instead_of_raising(harness, smi, answer):
    smi.answer = answer
    rec = harness.card()
    assert rec["name"] == "NVIDIA H100 80GB HBM3"
    assert rec["error"].startswith("nvidia-smi: ")
    assert "power_limit" not in rec


@pytest.mark.parametrize("timer, args", [("events_ms", (3, 1)), ("median_events_s", (3,)), ("median_wall_s", (3,)),
                                         ("graph_us", (3, 2))])
def test_timers_refuse_to_run_without_cuda(harness, monkeypatch, timer, args):
    monkeypatch.setattr(harness.torch.cuda, "is_available", lambda: False)
    calls = []
    with pytest.raises(RuntimeError, match="CUDA"):
        getattr(harness, timer)(lambda: calls.append(1), *args)
    assert calls == []                                      # nothing was run, so nothing was timed on the host
