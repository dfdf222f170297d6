"""Time select_k against torch.topk(sorted=True) on the same device tensors (one GPU).

Workloads (rows x len, k) cover every layout of select_k and both sides of each switch:
  kNN slab      16384 x 100000, k in {16, 64, 256, 1024}: pairwise_distance output, then select (one CTA per row)
  short rows    100000 x 1024, k = 32 and 1000000 x 128, k = 10 (whole rows sorted on chip); 100000 x 4096, k = 32
                (just above that switch: one CTA per row)
  long rows     16 x 2^24, k = 256 and 1 x 2^28, k = 1024 (rows split over CTAs)
  large k       100 x 100000, k = 50000 (segmented radix sort)
  all equal     16384 x 100000, k = 64: no value digit narrows anything
For each: the median of --runs calls of each (CUDA events, warm-up excluded), GB/s as rows * len * 4 / time, the card
and its power limit.  Every select_k output, the warm-up's included, is checked against torch.topk: values bit-equal,
indices equal wherever the value is unique in its row (topk's order among equal values is unspecified).  Exits non-zero
on a mismatch.  Prints one JSON line per workload.

  python scripts/select_k_time.py [--runs 10] [--only name,...]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from measure import card, time_ms  # noqa: E402
from raft_b200.common import DeviceResources  # noqa: E402
from raft_b200.matrix import select_k  # noqa: E402

WORKLOADS = [("slab", 16384, 100000, k, "normal") for k in (16, 64, 256, 1024)] + [
    ("short", 100000, 1024, 32, "normal"), ("short", 1000000, 128, 10, "normal"), ("short", 100000, 4096, 32, "normal"),
    ("long", 16, 2 ** 24, 256, "normal"), ("long", 1, 2 ** 28, 1024, "normal"),
    ("large_k", 100, 100000, 50000, "normal"), ("all_equal", 16384, 100000, 64, "equal")]


def mismatches(v, i, tv, ti):
    """values bit-equal everywhere; indices equal where the value occurs once in the row's selection"""
    bad = int((v.view(torch.int32) != tv.view(torch.int32)).sum())
    s = tv.view(torch.int32)
    unique = torch.ones_like(ti, dtype=torch.bool)
    unique[:, 1:] &= s[:, 1:] != s[:, :-1]
    unique[:, :-1] &= s[:, :-1] != s[:, 1:]
    return bad + int(((i != ti) & unique).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    gpu = card()
    h = DeviceResources()
    torch.manual_seed(7)
    failed = False
    for wname, rows, n, k, dist in WORKLOADS:
        if a.only and wname not in a.only.split(","):
            continue
        x = torch.randn((rows, n), device="cuda") if dist == "normal" else torch.full((rows, n), 0.5, device="cuda")
        outs = []
        t_sel = time_ms(lambda: outs.append(select_k(x, k=k, select_min=True, handle=h)), a.runs)
        t_top = time_ms(lambda: torch.topk(x, k, dim=1, largest=False, sorted=True), a.runs)
        tv, ti = torch.topk(x, k, dim=1, largest=False, sorted=True)
        bad = sum(mismatches(v, i, tv, ti) for v, i in outs)
        del outs, tv, ti
        med = statistics.median
        gbs = lambda t: round(rows * n * 4 / (t * 1e-3) / 1e9, 1)   # noqa: E731
        print(json.dumps({"workload": wname, "rows": rows, "len": n, "k": k, "data": dist,
                          "select_k_ms": round(med(t_sel), 3), "topk_ms": round(med(t_top), 3),
                          "select_k_GBps": gbs(med(t_sel)), "topk_GBps": gbs(med(t_top)),
                          "speedup": round(med(t_top) / med(t_sel), 2), "runs": a.runs, "mismatches": bad,
                          "card": gpu["name"], "power_limit": gpu["power_limit"]}), flush=True)
        failed |= bad != 0
        del x
        torch.cuda.empty_cache()
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
