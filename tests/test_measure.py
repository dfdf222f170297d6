"""scripts/measure.py, the timing scripts' one measuring module: no fallback without a device, the summary's keys, and a
clock sampler that leaves no thread behind when nvidia-smi is absent."""
import os
import sys
import threading
import time

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import measure  # noqa: E402


def test_card_and_time_ms_raise_without_a_device(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA device"):
        measure.card()
    calls = []
    with pytest.raises(RuntimeError, match="CUDA device"):
        measure.time_ms(lambda: calls.append(1), 3)
    assert calls == []


def test_summary_keys():
    s = measure.summary([2.00049, 1.0, 3.5])
    assert s == {"median": 2.0, "min": 1.0, "max": 3.5, "runs": [2.00049, 1.0, 3.5]}


def test_sm_clocks_without_nvidia_smi(monkeypatch, tmp_path):
    monkeypatch.setenv("PATH", str(tmp_path))
    assert measure.smi("clocks.sm", 0) is None
    raised = []
    monkeypatch.setattr(threading, "excepthook", raised.append)   # an exception in the sampling thread lands here
    before = set(threading.enumerate())
    with measure.SmClocks(0) as clk:
        time.sleep(0.5)   # a few polls
    assert raised == [] and clk.samples == []
    assert not clk._t.is_alive()
    assert set(threading.enumerate()) == before
