"""Time single_linkage (raft_b200.cluster.single_linkage) per stage, and the composition a user would write without it:
brute_force.knn, the graph copied to the host, scipy.sparse.csgraph.minimum_spanning_tree and a union-find dendrogram.

Stages come from one torch.profiler run of the call, cut at marker kernels in stream order: kNN (up to
sl_knn_edges_kernel), Borůvka (the rounds before the first connect), each connect round (sl_tree_min_init_kernel up to the
round's last Borůvka kernel, including its host synchronisation), and the dendrogram (the radix sort to the end of the
call: device sort and gather, copies, union-find on the host).  The total is CUDA events around the call (which
synchronises before it returns) after a warm-up, without the profiler, median of --reps.

Inputs: blobs with overlapping centres (a connected kNN graph: the baseline's MST is then the same spanning tree) and
blobs with separated centres (several kNN components: connect_components runs), at 100000 x 128 and 1000000 x 32, c = 15.
Prints one JSON line per measurement, and writes them to --out."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from measure import card, time_ms  # noqa: E402
from raft_b200.cluster import single_linkage  # noqa: E402
from raft_b200.neighbors import brute_force  # noqa: E402


def blobs(m, d, n_blobs, sep, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centers = (torch.rand((n_blobs, d), generator=g, device="cuda") * 2 - 1) * sep
    y = torch.randint(0, n_blobs, (m,), generator=g, device="cuda")
    return (centers[y] + torch.randn((m, d), generator=g, device="cuda")).contiguous()


def stages(x, c):
    """Per-stage times (ms) of one call from the profiler timeline."""
    from torch.profiler import ProfilerActivity, profile, record_function
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        with record_function("single_linkage_call"):
            out = single_linkage(x, 10, c=c)
    ev = prof.events()
    call = [e for e in ev if e.name == "single_linkage_call"][0]
    kern = sorted((e for e in ev if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    t0, t_end = call.time_range.start, call.time_range.end
    names = [k.name for k in kern]
    i_edges = max(i for i, n in enumerate(names) if "sl_knn_edges_kernel" in n)
    i_rounds = [i for i, n in enumerate(names) if "sl_tree_min_init_kernel" in n]
    i_sort = min(i for i, n in enumerate(names) if "DeviceRadixSort" in n)
    res = {"knn_ms": (kern[i_edges].time_range.end - t0) / 1e3}
    cuts = i_rounds + [i_sort]
    res["boruvka_ms"] = (kern[cuts[0]].time_range.start - kern[i_edges].time_range.end) / 1e3
    res["connect_rounds_ms"] = [(kern[b].time_range.start - kern[a].time_range.start) / 1e3 for a, b in zip(cuts, cuts[1:])]
    res["dendrogram_ms"] = (t_end - kern[i_sort].time_range.start) / 1e3
    res["n_connected_components"] = out.n_connected_components
    return res


def baseline(x, c):
    """brute_force.knn + scipy minimum_spanning_tree + a union-find dendrogram on the host (a connected kNN graph)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components, minimum_spanning_tree
    m = x.shape[0]
    nb = min(m, max(2, int(np.floor(np.log2(m))) + c))
    torch.cuda.synchronize()
    t = time.perf_counter()
    dist, idx = brute_force.knn(x, x, nb, metric="sqeuclidean")
    dist, idx = dist.cpu().numpy().ravel(), idx.cpu().numpy().ravel()
    t_knn = time.perf_counter()
    src = np.repeat(np.arange(m), nb)
    keep = src != idx
    # scipy drops explicit zeros: a tiny positive weight stands for a zero distance
    g = coo_matrix((np.maximum(dist[keep], np.float32(1e-30)), (src[keep], idx[keep])), shape=(m, m)).tocsr()
    T = minimum_spanning_tree(g).tocoo()
    t_mst = time.perf_counter()
    order = np.argsort(T.data, kind="stable")
    p = np.arange(m)

    def find(v):
        while p[v] != v:
            p[v] = p[p[v]]
            v = p[v]
        return v
    for a, b in zip(T.row[order], T.col[order]):
        ra, rb = find(a), find(b)
        p[rb] = ra
    t_end = time.perf_counter()
    ncomp = connected_components(g, directed=False)[0]
    return {"knn_ms": (t_knn - t) * 1e3, "mst_ms": (t_mst - t_knn) * 1e3, "dendrogram_ms": (t_end - t_mst) * 1e3,
            "total_ms": (t_end - t) * 1e3, "n_connected_components": int(ncomp)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="100000x128,1000000x32")
    ap.add_argument("--c", type=int, default=15)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-baseline", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    rows = []
    for shape in a.shapes.split(","):
        m, d = map(int, shape.split("x"))
        for kind, sep in (("overlapping", 1.0), ("separated", 200.0)):
            x = blobs(m, d, 10, sep, seed=m + d)
            r = {"shape": shape, "input": kind, "c": a.c, "card": gpu,
                 "total_ms": statistics.median(time_ms(lambda: single_linkage(x, 10, c=a.c), a.reps))}
            r.update(stages(x, a.c))
            rows.append(r)
            print(json.dumps(r), flush=True)
            if kind == "overlapping" and not a.no_baseline:
                b = {"shape": shape, "input": kind, "c": a.c, "card": gpu, "what": "baseline knn+scipy"}
                b.update(baseline(x, a.c))
                rows.append(b)
                print(json.dumps(b), flush=True)
            del x
            torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
