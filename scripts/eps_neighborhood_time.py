"""Time eps_neighbors_l2sq against the composition it replaces (one GPU).

Workloads (m x n x k, blobs data, eps = the squared distance that makes about 1 % of the pairs adjacent):
  100000 x 100000 x 128   the MMAs dominate
  1000000 x 8192 x 32     DBSCAN-like: the output dominates
  1000000 x 8190 x 32     the same with n % 16 != 0: adj leaves by the per-row copy instead of TMA
Arms: the fused call with adj, the fused call counting only, and the composition pairwise_distance(sqeuclidean) ->
torch.le -> sum(0).  Before any time is printed the fused adj / vd are checked equal to the composition's, bit for bit.
Median of --runs calls per arm (CUDA events, one warm-up call each).  Prints the card and its power limit, then one JSON
line per workload.

  python scripts/eps_neighborhood_time.py [--runs 5] [--only 0,1]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from measure import card, time_ms  # noqa: E402
from raft_b200.common import DeviceResources  # noqa: E402
from raft_b200.distance import pairwise_distance  # noqa: E402
from raft_b200.neighbors import eps_neighbors_l2sq  # noqa: E402

WORKLOADS = [(100000, 100000, 128), (1000000, 8192, 32), (1000000, 8190, 32)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    gpu = card()
    pl = "%s W, %s MHz" % (gpu["power_limit"], gpu["clocks_max_sm"])
    print("card: %s, power limit, max SM clock: %s" % (gpu["name"], pl), flush=True)
    h = DeviceResources()
    sel = [int(s) for s in a.only.split(",") if s] or range(len(WORKLOADS))
    for wi in sel:
        m, n, k = WORKLOADS[wi]
        c = oracle.make_blobs(16, k, seed=7)[2]
        x = torch.from_numpy(oracle.make_blobs(m, k, seed=11, centers=c)[0]).cuda()
        y = torch.from_numpy(oracle.make_blobs(n, k, seed=13, centers=c)[0]).cuda()
        dist = torch.empty((m, n), dtype=torch.float32, device="cuda")
        # eps from a sample of the distances: about 1 % adjacent
        pairwise_distance(x[:2048], y, out=dist[:2048], metric="sqeuclidean", handle=h)
        h.sync()
        eps = float(torch.quantile(dist[:2048, :4096].flatten().double(), 0.01))
        adj = torch.empty((m, n), dtype=torch.bool, device="cuda")
        vd = torch.empty(n + 1, dtype=torch.int64, device="cuda")

        def fused():
            eps_neighbors_l2sq(x, y, eps, adj=adj, vd=vd, handle=h)

        def count_only():
            eps_neighbors_l2sq(x, y, eps, vd=vd, return_adj=False, handle=h)

        def composition():
            pairwise_distance(x, y, out=dist, metric="sqeuclidean", handle=h)
            with torch.cuda.stream(h.torch_stream):
                ra = torch.le(dist, eps)
                # column sums over row slabs: a bool sum widens to int64, and the whole matrix at once does not fit
                cnt = torch.zeros(n, dtype=torch.int64, device="cuda")
                for r0 in range(0, m, 16384):
                    cnt += ra[r0:r0 + 16384].sum(0)
            return ra, cnt

        fused()
        h.sync()
        ra, cnt = composition()
        h.sync()
        assert torch.equal(adj, ra), "adj differs from the composition"
        assert torch.equal(vd[:n], cnt) and int(vd[n]) == int(cnt.sum()), "vd differs from the composition"
        frac = float(vd[n]) / (m * n)
        vd_adj = vd.clone()
        count_only()
        h.sync()
        assert torch.equal(vd, vd_adj), "count-only vd differs"
        del ra, cnt
        res = {}
        for arm, fn in (("fused_adj", fused), ("fused_count", count_only), ("composition", composition)):
            ts = time_ms(lambda: (fn(), h.sync()), a.runs)
            res[arm] = {"median_ms": round(statistics.median(ts), 3), "ms": [round(t, 3) for t in ts]}
        print(json.dumps({"m": m, "n": n, "k": k, "eps": eps, "adjacent_fraction": round(frac, 5), "card": gpu["name"],
                          "power_limit_max_sm_clock": pl, **res}), flush=True)
        del x, y, dist, adj, vd
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
