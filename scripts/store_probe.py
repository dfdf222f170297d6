#!/usr/bin/env python
"""Which property of the flagship kernel's store pattern costs bandwidth: scripts/store_probe.cu writes the flagship's
100000 x 100000 fp32 result the way expanded_tc_kernel<resident, EPI_STORE, POST_CLAMP> does (no MMAs, no operand
loads), once per variant, and times every variant in one process:

  policy   L2 hint of the TMA stores: evict_first (the kernel's), evict_normal, none
  G        128 G bytes per row per TMA store: 1 (a 2-D 64 x 32 box, the kernel's earlier box), or 2 (the kernel's
           32 x 64 box) or 4 through a 3-D view {32, n / 32, m}
  P        pairs of 8 KB boxes in each warpgroup's ring (the kernel: 1, wait_group.read 0)
  chunk    x tiles per work item (the kernel: 32; 1 makes the CTAs sweep whole rows of tiles together)
  idle     clock cycles each warpgroup spins before staging a half, a stand-in for the MMA turn

and two references: torch fill_ of the same tensor and a row-major st.global.v4 sweep.  Variants are alternated,
`--runs` rounds of `--steps` launches each, timed with CUDA events.  Every variant's output is checked at sampled
entries (each value is a function of its row and column).  The card's name, power limit and SM clocks during the rounds
are read in the same call.  Compare a variant at idle 0 with the kernel's stores-only diagnostic build
(scripts/tc_breakdown.py) before reading anything into the others: the probe leaves out the kernel's operand loads and
waits, and on an H100 the 128-byte pattern ran 2 ms faster here than in that build (DESIGN.md section 5).

usage: python scripts/store_probe.py [--runs 3] [--steps 5] [--idle 3000] [--out FILE]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from measure import SmClocks, card, summary, time_ms  # noqa: E402
from raft_b200 import _build  # noqa: E402

M, N = 100_000, 100_000
POLICY = {"evict_first": 0, "evict_normal": 1, "none": 2}


def variants(idle):
    v = [("G1 evict_first", 1, 1, "evict_first", 32, 0),
         ("G1 evict_normal", 1, 1, "evict_normal", 32, 0),
         ("G1 no hint", 1, 1, "none", 32, 0),
         ("G2 evict_first", 2, 1, "evict_first", 32, 0),
         ("G2 evict_normal", 2, 1, "evict_normal", 32, 0),
         ("G4 evict_first", 4, 1, "evict_first", 32, 0),
         ("G4 evict_normal", 4, 1, "evict_normal", 32, 0),
         ("G1 evict_first P2", 1, 2, "evict_first", 32, 0),
         ("G1 evict_first P3", 1, 3, "evict_first", 32, 0),
         ("G1 evict_normal P2", 1, 2, "evict_normal", 32, 0),
         ("G1 evict_first chunk1", 1, 1, "evict_first", 1, 0),
         ("G2 evict_first P2", 2, 2, "evict_first", 32, 0)]
    if idle > 0:
        v += [(f"{name} idle{idle}", g, p, pol, ch, idle) for name, g, p, pol, ch, _ in
              (v[0], v[1], v[3], v[4], v[7])]
    return v


def build(out):
    cmd = [_build._nvcc(), "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler",
           "-fPIC", "-o", out, os.path.join(HERE, "store_probe.cu")]
    subprocess.run(cmd, check=True)
    L = ctypes.CDLL(out)
    L.probe_launch.restype = ctypes.c_int
    L.probe_launch.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                               ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p]
    return L


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--idle", type=int, default=3000, help="clock cycles of the idle variants (0: none)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    tmp = tempfile.TemporaryDirectory(prefix="store_probe_")
    L = build(os.path.join(tmp.name, "store_probe.so"))

    import torch
    assert torch.cuda.is_available(), "store_probe needs a GPU"
    dev = torch.device("cuda", 0)
    d = torch.empty(M, N, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    vs = variants(args.idle)

    def launch(v):
        _, g, p, pol, ch, idle = v
        rc = L.probe_launch(d.data_ptr(), M, N, N, g, p, POLICY[pol], ch, idle, stream)
        if rc:
            raise RuntimeError(f"probe_launch {v[0]}: error {rc}")

    # each variant once on a poisoned buffer, checked at sampled entries: value(r, c) = fl(r / 1024 + c)
    g = torch.Generator(device=dev).manual_seed(0)
    rs = torch.cat([torch.randint(0, M, (8192,), device=dev, generator=g), torch.full((64,), M - 1, device=dev)])
    cs = torch.cat([torch.randint(0, N, (8192,), device=dev, generator=g), torch.arange(N - 64, N, device=dev)])
    want = (rs.double() / 1024 + cs.double()).float()
    for v in vs:
        d.fill_(float("nan"))
        launch(v)
        bad = int((d[rs, cs] != want).sum())
        if bad:
            raise RuntimeError(f"{v[0]}: {bad} sampled entries wrong")
    torch.cuda.synchronize()

    arms = [(v[0], lambda v=v: launch(v)) for v in vs] + [
        ("fill_", lambda: d.fill_(1.0)),
        ("st.global.v4 sweep", lambda: L.probe_launch(d.data_ptr(), M, N, N, 0, 0, 0, 0, 0, stream))]
    times = {nm: [] for nm, _ in arms}
    gpu = card(dev)
    with SmClocks(gpu["uuid"]) as clk:
        for _ in range(args.runs):
            for nm, fn in arms:
                fn()   # one warm-up launch after the previous arm: after a whole warm-up pass, the idle arms ran slower
                times[nm].append(time_ms(lambda: [fn() for _ in range(args.steps)], 1, warmup=0)[0] / args.steps)
    gb = M * N * 4 / 1e9
    res = {"shape": f"{M}x{N} fp32 ({gb:.0f} GB)", "runs": args.runs, "steps_per_run": args.steps,
           "card": gpu["name"], "power_limit_w": gpu["power_limit"], "clocks_max_sm_mhz": gpu["clocks_max_sm"],
           "clocks_sm_mhz": {"min": min(clk.samples), "median": statistics.median(clk.samples),
                             "max": max(clk.samples)} if clk.samples else None,
           "ms": {nm: {**summary(t), "tb_s": round(gb / statistics.median(t), 3)} for nm, t in times.items()}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    tmp.cleanup()


if __name__ == "__main__":
    main()
