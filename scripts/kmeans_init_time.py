"""Time the k-means|| seeding (raft_b200.cluster.init_scalable) against greedy k-means++ (init_plus_plus) on blobs of
1 000 000 x 128 with spread 0.3, for n_clusters in {16, 256, 1024, 4096} (greedy up to 1024).  Per n_clusters: the
seeding times (CUDA events, median of 3), both seeding costs, and each seeding's converged fit (max_iter 300,
tol 1e-4) inertia and n_iter.  The split of the k-means|| seeding times the same work through the public calls that run
its kernels: the 9 draws (select_k of 1 x m keys at L rows) and the 8 arg-min passes of x against L rows (the rounds),
the arg-min of x against all C candidates with the weight sums (the weights pass), a weighted greedy k-means++ plus
Lloyd fit on C rows (the recluster), and the greedy k-means++ on C rows alone.  Prints one JSON line per measurement
and, with --out, writes them to that file."""
import argparse
import json
import os
import sys
from statistics import median

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import kmeans_ref  # noqa: E402
import kmeans_scalable_ref  # noqa: E402
from measure import card, time_ms  # noqa: E402
from raft_b200 import _lib  # noqa: E402
from raft_b200.cluster import (KMeansParams, cluster_cost, compute_new_centroids, fit, init_plus_plus,  # noqa: E402
                               init_scalable)
from raft_b200.common import DeviceResources  # noqa: E402
from raft_b200.distance import fused_l2_nn  # noqa: E402


def select_k_1xm(keys, n, h):
    L = _lib.lib()
    m = keys.numel()
    val = torch.empty(n, dtype=torch.float32, device="cuda")
    idx = torch.empty(n, dtype=torch.int64, device="cuda")
    ws = h.workspace(L.b2d_select_k_workspace_bytes(1, m, n))
    _lib.check(L.b2d_select_k(h.stream_ptr, keys.data_ptr(), m, None, 1, m, n, 1, val.data_ptr(), idx.data_ptr(),
                              ws.data_ptr(), ws.numel()))
    return idx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1000000)
    ap.add_argument("--k", type=int, default=128)
    ap.add_argument("--ncs", default="16,256,1024,4096")
    ap.add_argument("--greedy-max", type=int, default=1024)
    ap.add_argument("--f", type=float, default=2.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = [{"gpu": card()}]
    print(json.dumps(rows[0]), flush=True)
    x, _, _ = kmeans_ref.blobs(a.m, a.k, 64, seed=1, spread=0.3)
    xd = torch.from_numpy(x).cuda()
    h = DeviceResources()
    for nc in [int(s) for s in a.ncs.split(",")]:
        L, C = kmeans_scalable_ref.sizes(a.m, nc, a.f)
        r = {"n_clusters": nc, "L": L, "C": C}
        # a call whose result is used is its own warm-up: the calls are seeded, so every call returns the same result
        cs = init_scalable(xd, n_clusters=nc, oversampling_factor=a.f, seed=0, handle=h)
        r["scalable_ms"] = median(time_ms(
            lambda: init_scalable(xd, n_clusters=nc, oversampling_factor=a.f, seed=0, handle=h), a.reps, warmup=0))
        r["scalable_cost"] = cluster_cost(xd, cs, handle=h)
        # the split, through the public calls that run the same kernels
        keys = torch.rand(a.m, device="cuda")
        cand = xd[torch.randperm(a.m, device="cuda")[:C]].contiguous()
        r["draw_ms"] = median(time_ms(lambda: select_k_1xm(keys, L, h), a.reps))
        r["round_argmin_ms"] = median(time_ms(lambda: fused_l2_nn(xd, cand[:L], sqrt=False, handle=h), a.reps))
        r["rounds_ms_est"] = 9 * r["draw_ms"] + 8 * r["round_argmin_ms"]

        def weights_pass():
            lab, _ = fused_l2_nn(xd, cand, sqrt=False, handle=h)
            new = torch.empty_like(cand)
            wpc = torch.empty(C, dtype=torch.float32, device="cuda")
            compute_new_centroids(xd, cand, lab.to(torch.int32), new, weight_per_cluster=wpc, handle=h)
            return wpc
        wpc = weights_pass()
        r["weights_pass_ms"] = median(time_ms(weights_pass, a.reps, warmup=0))
        rp = KMeansParams(n_clusters=nc, max_iter=300, tol=1e-4, seed=0)
        r["recluster_ms"] = median(time_ms(lambda: fit(rp, cand, sample_weights=wpc, handle=h), a.reps))
        r["recluster_greedy_ms"] = median(time_ms(lambda: init_plus_plus(cand, n_clusters=nc, seed=0, handle=h),
                                                  a.reps))
        fs = fit(KMeansParams(n_clusters=nc, seed=0, oversampling_factor=a.f), xd, handle=h)
        r["scalable_fit_inertia"], r["scalable_fit_n_iter"] = fs.inertia, fs.n_iter
        if nc <= a.greedy_max:
            cg = init_plus_plus(xd, n_clusters=nc, seed=0, handle=h)
            r["greedy_ms"] = median(time_ms(lambda: init_plus_plus(xd, n_clusters=nc, seed=0, handle=h), a.reps,
                                            warmup=0))
            r["greedy_cost"] = cluster_cost(xd, cg, handle=h)
            fg = fit(KMeansParams(n_clusters=nc, seed=0), xd, handle=h)
            r["greedy_fit_inertia"], r["greedy_fit_n_iter"] = fg.inertia, fg.n_iter
            r["fit_inertia_ratio"] = fs.inertia / fg.inertia
            r["seeding_speedup"] = r["greedy_ms"] / r["scalable_ms"]
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
