"""How the timing scripts here measure: the card that ran the work (queried by the uuid of torch's device, so the card
described is the card that ran), CUDA events around each call after warm-up, one summary of the times, and SM clock
samples during a run.  Without a CUDA device card() and time_ms() raise; there is no host-clock fallback."""
from __future__ import annotations

import statistics
import subprocess
import threading

import torch


def smi(query, gpu):
    """`nvidia-smi --query-gpu=<query>` of one card (an index or a GPU-<uuid>) as a list of strings, without units;
    None when nvidia-smi is missing or fails."""
    try:
        res = subprocess.run(["nvidia-smi", f"--id={gpu}", f"--query-gpu={query}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
    except (OSError, subprocess.TimeoutExpired):
        return None
    return [v.strip() for v in res.stdout.strip().split(",")] if res.returncode == 0 else None


def card(device=None) -> dict:
    """name, power_limit (W), clocks_max_sm (MHz) and uuid (GPU-...) of the card torch runs `device` on (default: the
    current device).  A field nvidia-smi cannot give is "unknown"."""
    if not torch.cuda.is_available():
        raise RuntimeError("measure.card needs a CUDA device")
    uuid = "GPU-" + str(torch.cuda.get_device_properties(device).uuid)
    fields = smi("name,power.limit,clocks.max.sm", uuid) or ["unknown"] * 3
    res = {k: "unknown" if v.startswith("[") else v for k, v in zip(("name", "power_limit", "clocks_max_sm"), fields)}
    res["uuid"] = uuid
    return res


def time_ms(fn, runs, warmup=1, stream=None) -> list[float]:
    """Milliseconds of each of `runs` calls of fn, between CUDA events recorded on `stream` (default: the current
    stream), after `warmup` calls and a device synchronise.  Time a loop by passing a fn that runs it."""
    if not torch.cuda.is_available():
        raise RuntimeError("measure.time_ms needs a CUDA device")
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def summary(ts) -> dict:
    """median, min and max of the times, rounded to 3 decimals, and the times under runs"""
    return {"median": round(statistics.median(ts), 3), "min": round(min(ts), 3), "max": round(max(ts), 3), "runs": ts}


class SmClocks:
    """SM clock samples (MHz) of card `gpu` (an nvidia-smi id), taken every 0.2 s while the block runs.  The sampling
    thread is stopped and joined when the block ends."""

    def __init__(self, gpu):
        self.gpu, self.samples, self._stop = gpu, [], threading.Event()

    def __enter__(self):
        def loop():
            while not self._stop.wait(0.2):
                v = smi("clocks.sm", self.gpu)
                if v and v[0].isdigit():
                    self.samples.append(int(v[0]))
        self._t = threading.Thread(target=loop, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join()
