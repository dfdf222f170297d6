"""Time masked_l2_nn against fused_l2_nn on the same data (one GPU).

Patterns (m = n = 262144, k = 64 by default; x sorted by group):
  cc      connect_components: 64 groups, adj[i, g] = colour(i) != g
  sparse  256 groups of 1024 rows; each 64-row slab of x is adjacent to 8 random groups
  worst   groups of 16 rows, adjacency random with p = 0.5: every tile is PARTIAL
For each pattern: the share of live tiles (from the pattern), the median of --runs times of each call (CUDA events
around the call, after a warm-up call), the card and its power limit.  Every masked_l2_nn call, the warm-up included, is
checked against an fp64 re-evaluation of a sample of rows.  Prints one JSON line per pattern.

  python scripts/masked_nn_time.py [--m 262144] [--n 262144] [--k 64] [--runs 5] [--patterns cc,sparse,worst]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from measure import card, time_ms  # noqa: E402
from raft_b200 import _lib  # noqa: E402
from raft_b200.common import DeviceResources  # noqa: E402
from raft_b200.distance import fused_l2_nn, masked_l2_nn  # noqa: E402


def pattern(kind, m, n, dev, gen):
    """(adj uint8 [m, G] on the device, group size)"""
    if kind == "cc":
        G = 64
        colour = torch.arange(m, device=dev) * G // m
        adj = (colour[:, None] != torch.arange(G, device=dev)[None, :]).to(torch.uint8)
        return adj, n // G
    if kind == "sparse":
        G = n // 1024
        adj = torch.zeros((m, G), dtype=torch.uint8, device=dev)
        for s in range((m + 63) // 64):
            adj[64 * s:64 * s + 64, torch.randperm(G, generator=gen, device="cpu")[:8].to(dev)] = 1
        return adj, 1024
    G = n // 16
    adj = torch.empty((m, G), dtype=torch.uint8, device=dev)
    for r0 in range(0, m, 8192):
        adj[r0:r0 + 8192] = (torch.rand((min(8192, m - r0), G), device=dev) < 0.5).to(torch.uint8)
    return adj, 16


def live_share(adj, size, m, n):
    """share of (64-row slab, 128-column half) tiles with at least one adjacent pair (groups of `size` rows, n % size == 0)"""
    S, H = (m + 63) // 64, (n + 127) // 128
    G = adj.shape[1]
    anyg = torch.zeros((S, G), dtype=torch.bool, device=adj.device)
    for s0 in range(0, S, 512):
        blk = adj[64 * s0:64 * (s0 + 512)]
        rows = blk.shape[0] // 64 * 64
        anyg[s0:s0 + rows // 64] = blk[:rows].view(-1, 64, G).amax(1) != 0
    if size >= 128:
        live = anyg[:, (torch.arange(H, device=adj.device) * 128) // size]
    else:
        live = anyg.view(S, H, 128 // size).any(2)
    return float(live.float().mean())


def check(xd, yd, adj, size, gi, gv, rows):
    """fp64 re-evaluation of the sampled rows: distances within 1e-4, indices equal up to near-ties"""
    xs = xd[rows].double()
    n, G = yd.shape[0], adj.shape[1]
    grp = torch.arange(n, device=yd.device) // size
    free = grp >= G                                 # rows past the last group end: in no group, never a candidate
    grp = torch.where(free, torch.zeros_like(grp), grp)
    bad = 0
    for c0 in range(0, len(rows), 64):
        r = rows[c0:c0 + 64]
        d = torch.cdist(xs[c0:c0 + 64], yd.double()) ** 2
        ok = (adj[r][:, grp] != 0) & ~free[None, :]
        d = torch.where(ok, d, torch.full_like(d, float("inf")))
        rv, ri = d.min(1)
        g_i, g_v = gi[r].long(), gv[r].double()
        close = (g_v - rv).abs() <= 1e-4 * torch.clamp(rv, min=1.0)
        d_got = d.gather(1, g_i[:, None].clamp(0, yd.shape[0] - 1))[:, 0]
        same = (g_i == ri) | ((d_got - rv).abs() <= 1e-5 * torch.clamp(rv, min=1.0))
        none = torch.isinf(rv)                      # no candidate: index 0x7fffffff
        ok_row = torch.where(none, g_i == 0x7FFFFFFF, close & same)
        bad += int((~ok_row).sum())
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=262144)
    ap.add_argument("--n", type=int, default=262144)
    ap.add_argument("--k", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--patterns", default="cc,sparse,worst")
    a = ap.parse_args()
    if a.n % 1024 or a.m % 64:
        ap.error("--n must be a multiple of 1024 and --m of 64 (the patterns' group sizes and 64-row slabs)")
    dev = torch.device("cuda:0")
    gpu = card(dev)
    gen = torch.Generator().manual_seed(7)
    torch.manual_seed(7)
    m, n, k = a.m, a.n, a.k
    xd = torch.randn((m, k), device=dev)
    yd = torch.randn((n, k), device=dev)
    h = DeviceResources()
    L = _lib.lib()
    rows = torch.randperm(m, generator=gen)[:256].to(dev)
    for kind in a.patterns.split(","):
        adj, size = pattern(kind, m, n, dev, gen)
        gidx = torch.arange(size, n + 1, size, dtype=torch.int32, device=dev)
        share = live_share(adj, size, m, n)
        outs = []
        t_mask = time_ms(lambda: outs.append(masked_l2_nn(xd, yd, adj, gidx, handle=h)), a.runs)
        bad = sum(check(xd, yd, adj, size, gi, gv, rows) for gi, gv in outs)
        _lib.check(L.b2d_set_option(b"nn_screen", 0.0))
        try:
            t_exact = time_ms(lambda: fused_l2_nn(xd, yd, sqrt=False, handle=h), a.runs)
        finally:
            _lib.check(L.b2d_set_option(b"nn_screen", 1.0))
        t_default = time_ms(lambda: fused_l2_nn(xd, yd, sqrt=False, handle=h), a.runs)
        med = statistics.median
        print(json.dumps({"pattern": kind, "m": m, "n": n, "k": k, "groups": int(adj.shape[1]), "live_tile_share": round(share, 4),
                          "masked_ms": round(med(t_mask), 3), "exact_fused_ms": round(med(t_exact), 3),
                          "default_fused_ms": round(med(t_default), 3),
                          "masked_over_exact": round(med(t_mask) / med(t_exact), 3),
                          "runs": a.runs, "masked_ms_all": [round(t, 3) for t in t_mask],
                          "sample_mismatches": bad, "card": gpu["name"], "power_limit": gpu["power_limit"]}),
              flush=True)
        del adj
        torch.cuda.empty_cache()
        if bad:
            sys.exit(1)


if __name__ == "__main__":
    main()
