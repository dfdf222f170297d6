"""Time neighbors.ball_cover against the brute-force entry points on the same points (one GPU, metric sqeuclidean).

Shapes (n x d): 1000000 x 2 uniform, 1000000 x 3 make_blobs (the clustered, slow case: dense balls) and 10000000 x 2
uniform.  Arms:
  build           build_index with the default ceil(sqrt(n)) landmarks
  all_knn         all_knn_query with k = 16, every row of the dataset a query
  knn / bf_knn    k = 16 for the first Q rows of the dataset, ball cover against brute_force.knn
  eps / bf_radius eps_nn against radius_neighbors for the same Q queries, eps chosen for about 16 neighbours per row
The brute-force arms do all Q x n pairs, so Q is a slice of the dataset (100000 at 10^6 rows, 10000 at 10^7) rather than
all of it; the ball-cover arms are timed on the same slice.  Before any time is printed, the two arms are checked to
agree up to the expanded / unexpanded difference: kNN distances within 1e-6 (|q|^2 + max |x|^2) (the expanded form's
error scales with the squared norms), every row brute force returns within that of the ball cover's k-th distance when
measured exactly (indices differ only among such near-ties; the share of equal indices is printed), and radius_neighbors'
pair count between the ball cover's at eps -/+ that tolerance.  Median of --runs calls per arm (CUDA events, one warm-up call each).  Prints the card and
its power limit, then one JSON line per shape.

  python scripts/ball_cover_time.py [--runs 3] [--only 0,1,2]
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
from raft_b200.neighbors import ball_cover, brute_force, radius_neighbors  # noqa: E402

SHAPES = [(1000000, 2, "uniform", 100000), (1000000, 3, "blobs", 100000), (10000000, 2, "uniform", 10000)]
K = 16


def points(n, d, kind):
    if kind == "uniform":
        return torch.rand((n, d), generator=torch.Generator("cuda").manual_seed(n + d), device="cuda")
    x, _, _ = oracle.make_blobs(n, d, seed=n + d)
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    c = card()
    print("card", c["name"], "power limit", c["power_limit"], "W", flush=True)
    sel = [int(v) for v in a.only.split(",")] if a.only else range(len(SHAPES))
    for si in sel:
        n, d, kind, nq = SHAPES[si]
        x = points(n, d, kind)
        q = x[:nq].contiguous()
        index = ball_cover.build_index(x, metric="sqeuclidean")
        # agreement of the arms
        bd, bi = ball_cover.knn_query(index, q, K)
        fd, fi = brute_force.knn(x, q, K, metric="sqeuclidean")
        # the expanded form's error is relative to the squared norms
        tol = 1e-6 * ((q * q).sum(1, keepdim=True) + (x * x).sum(1).max())
        assert ((bd - fd).abs() <= tol).all(), (bd[:2], fd[:2])
        # the rows brute force returns, measured as the ball cover measures, are within that of the k-th distance
        t = q[:, None, :] - x[fi]
        exact = (t[..., 0] * t[..., 0] + t[..., 1] * t[..., 1]) + (t[..., 2] * t[..., 2] if d == 3 else 0)
        assert (exact <= bd[:, -1:] + tol).all()
        same_idx = float((bi == fi).float().mean())
        del t, exact
        scale = float(bd[:, -1].median())
        eps = scale
        nnz_b = int(ball_cover.eps_nn(index, q, eps)[0][-1])
        nnz_r = int(radius_neighbors(x, q, eps, metric="sqeuclidean")[0][-1])
        tg = float(tol.max())
        lo, hi = (int(ball_cover.eps_nn(index, q, e)[0][-1]) for e in (eps - tg, eps + tg))
        assert lo <= nnz_r <= hi, (lo, nnz_r, hi)
        del bd, bi, fd, fi
        res = {"n": n, "d": d, "data": kind, "k": K, "queries": nq, "landmarks": int(np.ceil(np.sqrt(n))),
               "knn_same_index": round(same_idx, 5), "eps": eps, "eps_pairs": nnz_b, "radius_pairs": nnz_r,
               "card": c["name"], "power_limit_w": c["power_limit"]}
        arms = {
            "build": lambda: ball_cover.build_index(x, metric="sqeuclidean"),
            "all_knn": lambda: ball_cover.all_knn_query(index, K),
            "knn": lambda: ball_cover.knn_query(index, q, K),
            "bf_knn": lambda: brute_force.knn(x, q, K, metric="sqeuclidean"),
            "eps": lambda: ball_cover.eps_nn(index, q, eps),
            "bf_radius": lambda: radius_neighbors(x, q, eps, metric="sqeuclidean"),
        }
        for name, fn in arms.items():
            res[name + "_ms"] = summary(time_ms(fn, a.runs))["median"]
        print(json.dumps(res), flush=True)
        del index, x, q
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
