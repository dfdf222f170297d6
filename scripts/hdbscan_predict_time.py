"""Time HDBSCAN's approximate_predict on the random ball cover (one GPU, metric euclidean, min_samples = 10,
min_cluster_size = 50).

Fitted shapes (m x d): 1000000 x 2 uniform, 1000000 x 3 make_blobs and 10000000 x 2 uniform; queries: Q = 100000 and
1000000 points from the same distribution.  Arms:
  predict      cluster.approximate_predict: median of --runs calls (CUDA events, one warm-up call)
  model        cluster.hdbscan_model against cluster.hdbscan on the same points: the model's overhead
  composition  what a user could write without this call: ball_cover.knn_query with k = 2 min_samples, a torch gather
               of the fitted core distances and an arg-min of the mutual reachability over those k rows, then the
               condensed-tree walk in numpy (the tree taken from the fit's edges by tests/hdbscan_predict_ref.py outside
               the timing).  Its answers may differ by construction (k candidates only); the count of differing labels
               is reported.  Run where m <= --tree-rows, since the numpy condensing pass is slow.
  refit        cluster.hdbscan on the fitted and query rows together (Q = 100000 only)
Before timing, predicting a sample of 10000 fitted rows must return the fit's labels (the identity property; the
count of differences is printed, and uniform data may hold a duplicate row).  The largest depth of the condensed tree
(the parent walk's bound) is reported where the tree is exported.  Prints the card and its power limit, then one JSON
line per shape.

  python scripts/hdbscan_predict_time.py [--runs 3] [--only 0,1,2] [--tree-rows 1000000]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
from measure import card, summary, time_ms  # noqa: E402
from raft_b200.cluster import approximate_predict, hdbscan, hdbscan_model  # noqa: E402
from raft_b200.neighbors import ball_cover  # noqa: E402

SHAPES = [(1000000, 2, "uniform"), (1000000, 3, "blobs"), (10000000, 2, "uniform")]
QUERIES = [100000, 1000000]
METRIC, MIN_SAMPLES, MIN_CLUSTER_SIZE = "euclidean", 10, 50


def points(n, d, kind, seed, centers=None):
    if kind == "uniform":
        return torch.rand((n, d), generator=torch.Generator("cuda").manual_seed(seed), device="cuda"), None
    x, _, c = oracle.make_blobs(n, d, seed=seed, centers=centers)
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda(), c


def kw():
    return dict(min_cluster_size=MIN_CLUSTER_SIZE, min_samples=MIN_SAMPLES, metric=METRIC)


def depth(tree):
    """the largest number of parent steps from a cluster to the root"""
    par, dep = tree["parent"], np.zeros(len(tree["parent"]), np.int64)
    for c in range(1, len(par)):   # a parent's id is below its child's
        dep[c] = dep[par[c]] + 1
    return int(dep.max())


class Composition:
    """the kNN + gather + arg-min + numpy-walk arm"""

    def __init__(self, x, model, tree):
        self.index = ball_cover.build_index(x, metric=METRIC)
        d, _ = ball_cover.all_knn_query(self.index, MIN_SAMPLES)
        self.core = d[:, -1].contiguous()   # the fitted rows' core distances (metric units)
        self.tree = tree

    def __call__(self, q):
        d, i = ball_cover.knn_query(self.index, q, 2 * MIN_SAMPLES)
        cq = d[:, MIN_SAMPLES - 1:MIN_SAMPLES]
        w = torch.maximum(torch.maximum(cq, self.core[i]), d)
        a = torch.argmin(w, dim=1, keepdim=True)   # the first of the distance-sorted neighbours at the smallest w
        j = torch.gather(i, 1, a)[:, 0].cpu().numpy()
        W = torch.gather(w, 1, a)[:, 0].double().cpu().numpy()
        t = self.tree
        with np.errstate(divide="ignore"):
            lam = np.minimum(np.where(W > 0, 1.0 / W, np.inf), t["row_lambda"][j])
        p = t["row_parent"][j]
        while True:
            up = (p != 0) & (t["birth"][p] > lam)
            if not up.any():
                break
            p = np.where(up, t["parent"][p], p)
        o = t["owner"][p]
        lab = t["label"][o]
        lab = np.where((o == 0) & ~(t["single_root"] & (lam >= t["thr"])), -1, lab)
        return lab


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default="")
    ap.add_argument("--tree-rows", type=int, default=1000000)
    a = ap.parse_args()
    c = card()
    print("card", c["name"], "power limit", c["power_limit"], "W", flush=True)
    sel = [int(v) for v in a.only.split(",")] if a.only else range(len(SHAPES))
    for si in sel:
        m, d, kind = SHAPES[si]
        x, centers = points(m, d, kind, m + d)
        res = {"m": m, "d": d, "data": kind, "metric": METRIC, "min_samples": MIN_SAMPLES,
               "min_cluster_size": MIN_CLUSTER_SIZE, "card": c["name"], "power_limit_w": c["power_limit"]}
        model = hdbscan_model(x, **kw())
        res["n_clusters"] = model.output.n_clusters
        res["model_mb"] = round(model.buffer.numel() / 2 ** 20, 1)
        sample = torch.randperm(m, generator=torch.Generator().manual_seed(1))[:10000].cuda()
        p = approximate_predict(model, x[sample])
        res["identity_mismatches"] = int((p.labels != model.output.labels[sample]).sum())
        assert res["identity_mismatches"] <= 2, res
        res["hdbscan_ms"] = summary(time_ms(lambda: hdbscan(x, **kw()), a.runs))["median"]
        res["hdbscan_model_ms"] = summary(time_ms(lambda: hdbscan_model(x, **kw()), a.runs))["median"]
        comp = None
        if m <= a.tree_rows:
            import hdbscan_predict_ref as R
            mst = model.output.mst
            tree = R.export(mst.src.cpu().numpy(), mst.dst.cpu().numpy(), mst.weights.cpu().numpy(), m,
                            MIN_CLUSTER_SIZE)
            res["tree_depth"] = depth(tree)
            res["tree_clusters"] = len(tree["parent"])
            comp = Composition(x, model, tree)
        for nq in QUERIES:
            q, _ = points(nq, d, kind, 7 * m + nq, centers)
            r = {}
            r["predict_ms"] = summary(time_ms(lambda: approximate_predict(model, q), a.runs))["median"]
            if comp is not None:
                want = approximate_predict(model, q).labels.cpu().numpy()
                r["composition_ms"] = summary(time_ms(lambda: comp(q), a.runs))["median"]
                r["composition_label_differences"] = int((comp(q) != want).sum())
            if nq == QUERIES[0]:
                xq = torch.cat([x, q]).contiguous()
                r["refit_ms"] = summary(time_ms(lambda: hdbscan(xq, **kw()), a.runs))["median"]
                del xq
            res["q%d" % nq] = r
            del q
        print(json.dumps(res), flush=True)
        del x, model, comp
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
