#!/usr/bin/env python
"""Where the flagship kernel's time goes: expanded_tc_kernel<resident, EPI_STORE, POST_CLAMP> at L2Expanded
100000 x 100000 x 128 fp32, timed as built and in the three diagnostic builds of expanded_tc.cuh (B2D_TC_DIAG):

  as built      the library of this tree (raft_b200/libraft_b200.so)
  MMAs only     B2D_TC_DIAG=1: no epilogue and no staging, the accumulators kept live
  stores out    B2D_TC_DIAG=2: every value computed and staged in shared memory, no TMA store issued
  stores only   B2D_TC_DIAG=3: no MMAs (zeros are computed on and staged), TMA stores on

All four libraries are loaded into one process and timed alternately, `--runs` rounds of `--steps` calls each, with the
kernel's own CUDA events (b2d_profile_begin / b2d_profile_end: operand preparation is not in the figure).  The card's
name, power limit and SM clocks during the timed rounds are read in the same call.  Only the as-built figures are
results; the diagnostic builds compute wrong distances by design.

usage: python scripts/tc_breakdown.py [--lib-dir DIR] [--as-built LIB] [--runs 3] [--steps 10] [--out FILE] [--build-only]
  --lib-dir:  where the diagnostic libraries are built, or found if they are newer than every source (default: a
              temporary directory)
  --as-built: time this library as the "as built" variant instead of the tree's (with --lib-dir holding diagnostic
              builds of the same sources: how an earlier version of the kernel is measured)
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from measure import SmClocks, card, summary  # noqa: E402
from raft_b200 import _build  # noqa: E402

M, N, K = 100_000, 100_000, 128
VARIANTS = [("as built", None), ("MMAs only", 1), ("stores out", 2), ("stores only", 3)]


def lib_path(lib_dir, diag, as_built=None):
    if diag is None:
        return as_built or _build.SO_PATH
    return os.path.join(lib_dir, f"diag{diag}", "libraft_b200.so")


def build_variants(lib_dir):
    """nvcc of the whole library once per diagnostic switch, in parallel; up-to-date libraries are kept."""
    _build.build()
    units = [s for s in _build.sources() if s.endswith(".cu")]
    newest = max(os.path.getmtime(s) for s in _build.sources())
    procs = []
    for _, diag in VARIANTS:
        out = lib_path(lib_dir, diag)
        if diag is None or (os.path.exists(out) and os.path.getmtime(out) > newest):
            continue
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cmd = [_build._nvcc()] + _build.NVCC_FLAGS + [f"-DB2D_TC_DIAG={diag}", "-o", out] + units + ["-ldl"]
        procs.append((diag, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for diag, pr in procs:
        log = pr.communicate()[0]
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed for B2D_TC_DIAG={diag}:\n{log}")


def load(path):
    L = ctypes.CDLL(path)
    i64, vp, sz, ci, cf = ctypes.c_int64, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_float
    L.b2d_last_error.restype = ctypes.c_char_p
    L.b2d_pairwise_workspace_bytes.restype = sz
    L.b2d_pairwise_workspace_bytes.argtypes = [ci, ci, i64, i64, i64]
    L.b2d_pairwise_distance.restype = ci
    L.b2d_pairwise_distance.argtypes = [vp, ci, ci, vp, i64, vp, i64, vp, i64, i64, i64, i64, ci, cf, vp, sz]
    L.b2d_profile_begin.restype = ci
    L.b2d_profile_begin.argtypes = [ci]
    L.b2d_profile_end.restype = ci
    L.b2d_profile_end.argtypes = [vp, ci, vp]
    return L


def check(L, rc):
    if rc != 0:
        raise RuntimeError(L.b2d_last_error().decode("utf-8", "replace"))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib-dir", default=None)
    ap.add_argument("--as-built", default=None)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    ap.add_argument("--build-only", action="store_true")
    args = ap.parse_args()
    tmp = None
    if args.lib_dir is None:
        tmp = tempfile.TemporaryDirectory(prefix="tc_breakdown_")
        args.lib_dir = tmp.name
    if args.as_built is None:
        build_variants(args.lib_dir)
    if args.build_only:
        return

    import torch
    assert torch.cuda.is_available(), "tc_breakdown needs a GPU"
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(M, K, device=dev, generator=g) * 3
    y = torch.randn(N, K, device=dev, generator=g) * 3
    out = torch.empty(M, N, device=dev)
    libs = [(name, load(lib_path(args.lib_dir, diag, args.as_built))) for name, diag in VARIANTS]
    ws_bytes = max(L.b2d_pairwise_workspace_bytes(0, 0, M, N, K) for _, L in libs)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def call(L):
        check(L, L.b2d_pairwise_distance(stream, 0, 0, x.data_ptr(), K, y.data_ptr(), K, out.data_ptr(), N, M, N, K, 1,
                                         2.0, ws.data_ptr(), ws_bytes))

    for _, L in libs:   # module load, function attributes, tensor maps
        call(L)
        call(L)
    torch.cuda.synchronize()
    gpu = card(dev)
    times = {name: [] for name, _ in libs}
    with SmClocks(gpu["uuid"]) as clk:
        for _ in range(args.runs):
            for name, L in libs:
                call(L)   # one warm-up call after the previous variant
                check(L, L.b2d_profile_begin(args.steps))
                for _ in range(args.steps):
                    call(L)
                buf = (ctypes.c_float * args.steps)()
                cnt = ctypes.c_int(0)
                check(L, L.b2d_profile_end(buf, args.steps, ctypes.byref(cnt)))
                times[name].append(sum(buf[i] for i in range(cnt.value)) / max(1, cnt.value))
    res = {"kernel": "expanded_tc_kernel<resident, EPI_STORE, POST_CLAMP>",
           "shape": f"L2Expanded {M}x{N}x{K} fp32", "runs": args.runs, "steps_per_run": args.steps,
           "card": gpu["name"], "power_limit_w": gpu["power_limit"], "clocks_max_sm_mhz": gpu["clocks_max_sm"],
           "clocks_sm_mhz": {"min": min(clk.samples), "median": statistics.median(clk.samples),
                             "max": max(clk.samples)} if clk.samples else None,
           "kernel_ms": {name: summary(v) for name, v in times.items()}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
