"""Time HDBSCAN on the random ball cover (one GPU, metric euclidean, min_samples = 10, min_cluster_size = 50).

Shapes (m x d): 1000000 x 2 uniform, 1000000 x 3 make_blobs and 10000000 x 2 uniform.  Arms:
  hdbscan   cluster.hdbscan: median of --runs calls (CUDA events, one warm-up call)
  split     one torch.profiler run of the call: device milliseconds of the index build (bc_* kernels and the build's
            sorts), the core distances (hdb_core / hdb_cmin), the Borůvka rounds (sl_* / slr_* / hdb_walk kernels; the
            walk on its own as well) and the edge sort; the host tree stages taken as hdbscan minus those
  emst      cluster.emst on the same points: the floor the mutual-reachability rounds are compared with
  sklearn   sklearn.cluster.HDBSCAN on the CPU, one fit of the first 100000 rows (the user's alternative), with the
            agreement of its labels with hdbscan's on those rows (adjusted Rand index; tied weights may merge
            differently)
Before timing, the arms are checked against each other: the mutual-reachability tree's sorted weights are at least the
EMST's, edge for edge (w >= s), and the tree's edges come in ascending weight with src < dst.  Prints the card and its
power limit, then one JSON line per shape.

  python scripts/hdbscan_rbc_time.py [--runs 3] [--only 0,1,2] [--no-sklearn]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from measure import card, summary, time_ms  # noqa: E402
from raft_b200.cluster import emst, hdbscan  # noqa: E402

SHAPES = [(1000000, 2, "uniform"), (1000000, 3, "blobs"), (10000000, 2, "uniform")]
METRIC, MIN_SAMPLES, MIN_CLUSTER_SIZE = "euclidean", 10, 50
SKLEARN_ROWS = 100000


def points(n, d, kind):
    if kind == "uniform":
        return torch.rand((n, d), generator=torch.Generator("cuda").manual_seed(n + d), device="cuda")
    x, _, _ = oracle.make_blobs(n, d, seed=n + d)
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def fit(x):
    return hdbscan(x, min_cluster_size=MIN_CLUSTER_SIZE, min_samples=MIN_SAMPLES, metric=METRIC)


def split(x):
    """device milliseconds of one call by stage, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fit(x)
        torch.cuda.synchronize()
    out = {k: 0.0 for k in ("build", "core", "rounds", "walk", "edge_sort", "rest")}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        name = e.key
        if "hdb_core" in name or "hdb_cmin" in name:
            g = "core"
        elif "bc_" in name:
            g = "build"
        elif "slr_" in name or "sl_" in name or "hdb_walk" in name:
            g = "rounds"
        elif "Radix" in name or "Onesweep" in name or "cub" in name:
            g = "build" if "unsigned long long" in name else "edge_sort"
        else:
            g = "rest"
        out[g] += us / 1000.0
        if "hdb_walk" in name:
            out["walk"] += us / 1000.0
    return {k: round(v, 3) for k, v in out.items()}


def check(o, e):
    w, s = o.mst.weights.cpu().numpy(), e.weights.cpu().numpy()
    assert (np.sort(w) >= np.sort(s)).all(), "the MR tree's weights fall below the EMST's"
    a, b = o.mst.src.cpu().numpy(), o.mst.dst.cpu().numpy()
    assert (a < b).all() and (np.diff(w) >= 0).all(), "edges out of order"


def sklearn_arm(x, ours):
    try:
        from sklearn.cluster import HDBSCAN
        from sklearn.metrics import adjusted_rand_score
    except ImportError:
        return None, None
    xs = x[:SKLEARN_ROWS].cpu().numpy()
    t0 = time.perf_counter()
    sk = HDBSCAN(min_cluster_size=MIN_CLUSTER_SIZE, min_samples=MIN_SAMPLES).fit(xs)
    ms = (time.perf_counter() - t0) * 1e3
    return round(ms, 1), round(float(adjusted_rand_score(sk.labels_, ours)), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default="")
    ap.add_argument("--no-sklearn", action="store_true")
    a = ap.parse_args()
    c = card()
    print("card", c["name"], "power limit", c["power_limit"], "W", flush=True)
    sel = [int(v) for v in a.only.split(",")] if a.only else range(len(SHAPES))
    for si in sel:
        m, d, kind = SHAPES[si]
        x = points(m, d, kind)
        res = {"m": m, "d": d, "data": kind, "metric": METRIC, "min_samples": MIN_SAMPLES,
               "min_cluster_size": MIN_CLUSTER_SIZE, "card": c["name"], "power_limit_w": c["power_limit"]}
        o, e = fit(x), emst(x, metric=METRIC)
        check(o, e)
        res["n_clusters"] = o.n_clusters
        res["noise_fraction"] = round(float((o.labels < 0).float().mean()), 4)
        del o, e
        res["hdbscan_ms"] = summary(time_ms(lambda: fit(x), a.runs))["median"]
        res["emst_ms"] = summary(time_ms(lambda: emst(x, metric=METRIC), a.runs))["median"]
        res["split_ms"] = split(x)
        dev = sum(v for k, v in res["split_ms"].items() if k != "walk")
        res["split_ms"]["host_tree"] = round(res["hdbscan_ms"] - dev, 3)
        if not a.no_sklearn and si == 0:
            sub = x[:SKLEARN_ROWS].contiguous()
            ours = fit(sub).labels.cpu().numpy()
            res["sklearn_rows"] = SKLEARN_ROWS
            res["sklearn_cpu_ms"], res["sklearn_ari"] = sklearn_arm(sub, ours)
            res["hdbscan_ms_at_sklearn_rows"] = summary(time_ms(lambda: fit(sub), a.runs))["median"]
        print(json.dumps(res), flush=True)
        del x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
