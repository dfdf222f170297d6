"""Time the exact single linkage on the random ball cover (one GPU, metric euclidean).

Shapes (m x d): 1000000 x 2 uniform, 1000000 x 3 make_blobs and 10000000 x 2 uniform.  Arms:
  emst        cluster.emst: median of --runs calls (CUDA events, one warm-up call)
  pairwise    single_linkage(linkage="pairwise", n_clusters=10): median of --runs calls; the EMST plus the host
              dendrogram
  split       one torch.profiler run of the pairwise call: device milliseconds of the index build (bc_* kernels and the
              build's sorts), the Borůvka rounds (sl_* / slr_* kernels; the walk on its own as well), the edge sort, and
              the host dendrogram taken as pairwise - emst
  knn_graph   single_linkage(linkage="knn_graph", c=15), one call; 10^6 rows only
  knn2        ball_cover.all_knn_query(k=2) on a built index: the floor of one round's walk (every row's nearest other
              row, without colours)
Prints the card and its power limit, then one JSON line per shape.

  python scripts/single_linkage_rbc_time.py [--runs 3] [--only 0,1,2]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from measure import card, summary, time_ms  # noqa: E402
from raft_b200.cluster import emst, single_linkage  # noqa: E402
from raft_b200.neighbors import ball_cover  # noqa: E402

SHAPES = [(1000000, 2, "uniform"), (1000000, 3, "blobs"), (10000000, 2, "uniform")]
METRIC, N_CLUSTERS = "euclidean", 10
KNN_GRAPH_MAX = 1000000


def points(n, d, kind):
    if kind == "uniform":
        return torch.rand((n, d), generator=torch.Generator("cuda").manual_seed(n + d), device="cuda")
    x, _, _ = oracle.make_blobs(n, d, seed=n + d)
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def split(x):
    """device milliseconds of one pairwise call by stage, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        single_linkage(x, N_CLUSTERS, metric=METRIC, linkage="pairwise")
        torch.cuda.synchronize()
    out = {k: 0.0 for k in ("build", "rounds", "walk", "edge_sort", "rest")}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        name = e.key
        if "bc_" in name:
            g = "build"
        elif "slr_" in name or "sl_" in name:
            g = "rounds"
        elif "Radix" in name or "Onesweep" in name or "cub" in name:
            # the build sorts (unsigned long long) keys; the edge sorts int and long long keys
            g = "build" if "unsigned long long" in name else "edge_sort"
        else:
            g = "rest"
        out[g] += us / 1000.0
        if "slr_walk" in name:
            out["walk"] += us / 1000.0
    return {k: round(v, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    c = card()
    print("card", c["name"], "power limit", c["power_limit"], "W", flush=True)
    sel = [int(v) for v in a.only.split(",")] if a.only else range(len(SHAPES))
    for si in sel:
        m, d, kind = SHAPES[si]
        x = points(m, d, kind)
        res = {"m": m, "d": d, "data": kind, "metric": METRIC, "n_clusters": N_CLUSTERS, "card": c["name"],
               "power_limit_w": c["power_limit"]}
        t = emst(x, metric=METRIC)
        res["longest_edge"] = float(t.weights[-1])
        res["emst_ms"] = summary(time_ms(lambda: emst(x, metric=METRIC), a.runs))["median"]
        res["pairwise_ms"] = summary(time_ms(lambda: single_linkage(x, N_CLUSTERS, metric=METRIC, linkage="pairwise"),
                                             a.runs))["median"]
        res["split_ms"] = split(x)
        res["split_ms"]["dendrogram_host"] = round(res["pairwise_ms"] - res["emst_ms"], 3)
        index = ball_cover.build_index(x, metric=METRIC)
        res["knn2_ms"] = summary(time_ms(lambda: ball_cover.all_knn_query(index, 2), a.runs))["median"]
        del index
        if m <= KNN_GRAPH_MAX:
            res["knn_graph_ms"] = summary(time_ms(lambda: single_linkage(x, N_CLUSTERS, metric=METRIC), 1,
                                                  warmup=0))["median"]
        else:
            res["knn_graph_ms"] = None
        print(json.dumps(res), flush=True)
        del x, t
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
