"""Time dbscan(algorithm="rbc") against the brute fit and against the composition a user can write today (one GPU, metric
euclidean, min_samples = 10).

Shapes (m x d): 1000000 x 2 uniform, 1000000 x 3 make_blobs and 10000000 x 2 uniform.  eps is the median distance to
the 30th neighbour over a sample of rows (ball_cover.knn_query), so a row has about 30 neighbours.  Arms:
  rbc          dbscan(algorithm="rbc"): median of --runs calls (CUDA events, one warm-up call), then one torch.profiler
               run for the time of the index build and of each walk (degree, link, border) and the rest
  brute        dbscan(algorithm="brute"), one call (a warm-up would double a multi-second arm); skipped at 10^7 rows,
               where its m^2 pairs per pass are out of reach
  composition  ball_cover.build_index + ball_cover.eps_nn on the device, then on the host scipy's connected components
               of the core rows and the border rule; one call.  Its labels are checked against the rbc fit's first.
Prints the card and its power limit, then one JSON line per shape.

  python scripts/dbscan_rbc_time.py [--runs 3] [--only 0,1,2]
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
from raft_b200.cluster import dbscan  # noqa: E402
from raft_b200.neighbors import ball_cover  # noqa: E402

SHAPES = [(1000000, 2, "uniform"), (1000000, 3, "blobs"), (10000000, 2, "uniform")]
METRIC, MIN_SAMPLES, NEIGHBOURS = "euclidean", 10, 30
BRUTE_MAX = 1000000


def points(n, d, kind):
    if kind == "uniform":
        return torch.rand((n, d), generator=torch.Generator("cuda").manual_seed(n + d), device="cuda")
    x, _, _ = oracle.make_blobs(n, d, seed=n + d)
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def pick_eps(x):
    index = ball_cover.build_index(x, metric=METRIC)
    sel = torch.randperm(x.shape[0], device="cuda", generator=torch.Generator("cuda").manual_seed(1))[:4096]
    dist, _ = ball_cover.knn_query(index, x[sel].contiguous(), NEIGHBOURS)
    return float(dist[:, -1].median())


def composition(x, eps):
    """eps_nn on the device, then the DBSCAN rules on the host: core rows, scipy components, the border rule"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    m = x.shape[0]
    index = ball_cover.build_index(x, metric=METRIC)
    indptr, indices, _ = ball_cover.eps_nn(index, x, eps)
    deg = (indptr[1:] - indptr[:-1]).cpu().numpy()
    rows = np.repeat(np.arange(m), deg)
    cols = indices.cpu().numpy()
    core = deg >= MIN_SAMPLES
    both = core[rows] & core[cols]
    g = coo_matrix((np.ones(int(both.sum()), np.int8), (rows[both], cols[both])), shape=(m, m))
    _, comp = connected_components(g, directed=True, connection="weak")
    cidx = np.flatnonzero(core)
    first = np.full(m, m, np.int64)
    np.minimum.at(first, comp[cidx], cidx)
    roots = first[comp[cidx]]
    uniq = np.unique(roots)
    labels = np.full(m, -1, np.int64)
    labels[cidx] = np.searchsorted(uniq, roots)
    hit = ~core[rows] & core[cols]
    best = np.full(m, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(best, rows[hit], labels[cols[hit]])
    nb = ~core & (best != np.iinfo(np.int64).max)
    labels[nb] = best[nb]
    return labels.astype(np.int32), int(uniq.size)


def walk_times(x, eps):
    """device milliseconds of one rbc fit by kernel group, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dbscan(x, eps, min_samples=MIN_SAMPLES, metric=METRIC, algorithm="rbc")
        torch.cuda.synchronize()
    groups = {"degree": "db_rbc_degree", "link": "db_rbc_link", "border": "db_rbc_border"}
    out = {k: 0.0 for k in ("build", "degree", "link", "border", "rest")}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        name = e.key
        g = next((k for k, v in groups.items() if v in name), None)
        if g is None:
            g = "build" if ("bc_" in name or "Radix" in name or "Onesweep" in name or "cub" in name) else "rest"
        out[g] += us / 1000.0
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
        eps = pick_eps(x)
        fit = dbscan(x, eps, min_samples=MIN_SAMPLES, metric=METRIC, algorithm="rbc")
        lab = fit.labels.cpu().numpy()
        res = {"m": m, "d": d, "data": kind, "metric": METRIC, "eps": eps, "min_samples": MIN_SAMPLES,
               "clusters": fit.n_clusters, "core": int(fit.core_sample_indices.numel()), "noise": int((lab == -1).sum()),
               "card": c["name"], "power_limit_w": c["power_limit"]}
        # the composition must give the fit's labels before anything is timed
        t0 = time.perf_counter()
        comp_lab, comp_nc = composition(x, eps)
        res["composition_ms"] = round(1000 * (time.perf_counter() - t0), 1)
        assert comp_lab.tobytes() == lab.tobytes() and comp_nc == fit.n_clusters, "composition disagrees with the fit"
        res["composition_agrees"] = True
        res["rbc_ms"] = summary(time_ms(lambda: dbscan(x, eps, min_samples=MIN_SAMPLES, metric=METRIC,
                                                       algorithm="rbc"), a.runs))["median"]
        res["rbc_profile_ms"] = walk_times(x, eps)
        if m <= BRUTE_MAX:
            res["brute_ms"] = summary(time_ms(lambda: dbscan(x, eps, min_samples=MIN_SAMPLES, metric=METRIC,
                                                             algorithm="brute"), 1, warmup=0))["median"]
        else:
            res["brute_ms"] = None
            res["brute_skipped"] = "m^2 = %.0e pairs per pass" % (float(m) * m)
        print(json.dumps(res), flush=True)
        del x, fit
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
