"""Time dbscan (raft_b200.cluster.dbscan) per pass, and two compositions a user would write without it:
  gpu+scipy  the public eps_neighbors_l2sq per column batch, torch.nonzero, the entries copied to the host,
             scipy.sparse.csgraph.connected_components over the core rows and the border rule in numpy;
  sklearn    sklearn.cluster.DBSCAN on the host cores, on the first --sk-rows rows (the GPU call is timed there too).

Passes come from one torch.profiler run of the call, cut at marker kernels in stream order: degrees (the call's start,
operand preparation included, to the end of db_core_kernel), links (to the end of db_compress_kernel), border (to the
first scan kernel after it) and numbering (the rest).  The total is CUDA events around the call after a warm-up,
median of --reps.

Inputs: Gaussian blobs of three spreads with 10 % uniform noise; eps is set from a row sample so that about --density of
the pairs are adjacent, which leaves core, border and noise points.  Shapes: 100000 x 128 (one 2^30-byte batch plan of
ten batches) and 1000000 x 32 (977 batches of 1024 columns).  Prints one JSON line per measurement (the card, its power
limit and max SM clock included) and writes them to --out."""
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
from raft_b200.cluster import dbscan  # noqa: E402
from raft_b200.neighbors.epsilon_neighborhood import eps_neighbors_l2sq  # noqa: E402


def blobs(m, d, n_blobs, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centers = (torch.rand((n_blobs, d), generator=g, device="cuda") * 2 - 1) * 20
    spread = torch.tensor([0.5, 1.0, 2.0], device="cuda")[torch.randint(0, 3, (n_blobs,), generator=g, device="cuda")]
    y = torch.randint(0, n_blobs, (m,), generator=g, device="cuda")
    x = centers[y] + spread[y, None] * torch.randn((m, d), generator=g, device="cuda")
    noise = torch.rand(m, generator=g, device="cuda") < 0.1
    x[noise] = (torch.rand((int(noise.sum()), d), generator=g, device="cuda") * 2 - 1) * 22
    return x.contiguous()


def pick_eps(x, density):
    s = x[torch.randperm(x.shape[0], device="cuda")[:4000]].double()
    d2 = torch.cdist(s, s).pow(2)
    return float(torch.quantile(d2[~torch.eye(len(s), dtype=torch.bool, device="cuda")][:10 ** 7], density).sqrt())


def passes(x, eps, ms):
    """Per-pass times (ms) of one call from the profiler timeline."""
    from torch.profiler import ProfilerActivity, profile, record_function
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        with record_function("dbscan_call"):
            out = dbscan(x, eps, min_samples=ms)
    ev = prof.events()
    kern = sorted((e for e in ev if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    names = [k.name for k in kern]
    first = min(i for i, n in enumerate(names) if "prep_max_kernel" in n)
    i_core = max(i for i, n in enumerate(names) if "db_core_kernel" in n)
    i_comp = max(i for i, n in enumerate(names) if "db_compress_kernel" in n)
    i_scan = min(i for i, n in enumerate(names) if "km_scan_tiles_kernel" in n and i > i_comp)
    i_last = max(i for i, n in enumerate(names) if "db_label_kernel" in n)
    t = [kern[first].time_range.start, kern[i_core].time_range.end, kern[i_comp].time_range.end,
         kern[i_scan].time_range.start, kern[i_last].time_range.end]
    res = {"device_span_ms": (t[4] - t[0]) / 1e3}
    for name, a, b in zip(("degrees", "links", "border", "numbering"), t, t[1:]):
        res[name + "_ms"] = (b - a) / 1e3
    res["launches"] = len([n for n in names[first:i_last + 1]])
    res["eps_launches"] = len([n for n in names[first:i_last + 1] if "expanded_tc_kernel" in n])
    res["n_clusters"] = out.n_clusters
    lab = out.labels
    res["core"] = int(out.core_sample_indices.numel())
    res["noise"] = int((lab == -1).sum())
    res["border"] = int(lab.numel() - res["core"] - res["noise"])
    return res, out


def composition(x, eps, ms, max_bytes=1 << 30):
    """public eps_neighbors_l2sq per column batch + torch.nonzero + scipy connected components + the border rule"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    m = x.shape[0]
    b = min(m, max(256, max_bytes // m // 256 * 256))
    e = float(np.float32(np.float64(eps) ** 2))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rows, cols = [], []
    for s in range(0, m, b):
        adj, _ = eps_neighbors_l2sq(x, x[s:s + b], e)
        nz = torch.nonzero(adj)
        rows.append(nz[:, 0].cpu().numpy())
        cols.append((nz[:, 1] + s).cpu().numpy())
        del adj, nz
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    t1 = time.perf_counter()
    core = np.bincount(cols, minlength=m) >= ms
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
    t2 = time.perf_counter()
    return {"eps_nonzero_copy_ms": (t1 - t0) * 1e3, "host_components_border_ms": (t2 - t1) * 1e3,
            "total_ms": (t2 - t0) * 1e3, "entries": int(rows.size)}, labels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="100000x128,1000000x32")
    ap.add_argument("--density", default="0.01,0.0005", help="adjacent fraction of the pairs, per shape")
    ap.add_argument("--min-samples", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sk-rows", type=int, default=10000)
    ap.add_argument("--no-baseline", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    rows = []

    def emit(r):
        r["card"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)

    for shape, dens in zip(a.shapes.split(","), map(float, a.density.split(","))):
        m, d = map(int, shape.split("x"))
        x = blobs(m, d, max(10, m // 1000), seed=m + d)
        eps = pick_eps(x, dens)
        r = {"shape": shape, "eps": eps, "min_samples": a.min_samples, "what": "dbscan",
             "total_ms": statistics.median(time_ms(lambda: dbscan(x, eps, min_samples=a.min_samples), a.reps))}
        p, out = passes(x, eps, a.min_samples)
        r.update(p)
        emit(r)
        if not a.no_baseline and m <= 200000:
            c, lab = composition(x, eps, a.min_samples)
            c.update({"shape": shape, "what": "baseline eps_neighbors per batch + nonzero + scipy",
                      "labels_equal": bool((lab == out.labels.cpu().numpy()).all())})
            emit(c)
        if not a.no_baseline and a.sk_rows and m <= 200000:
            from sklearn.cluster import DBSCAN
            xs = x[:a.sk_rows].contiguous()
            xh = xs.cpu().numpy().astype(np.float64)
            t = time.perf_counter()
            sk = DBSCAN(eps=eps, min_samples=a.min_samples, n_jobs=-1).fit(xh)
            t_sk = (time.perf_counter() - t) * 1e3
            o = dbscan(xs, eps, min_samples=a.min_samples)
            emit({"shape": "%dx%d" % (a.sk_rows, d), "what": "sklearn.cluster.DBSCAN n_jobs=-1 (host)",
                  "cpus": os.cpu_count(), "total_ms": t_sk,
                  "gpu_total_ms": statistics.median(time_ms(lambda: dbscan(xs, eps, min_samples=a.min_samples),
                                                            a.reps)),
                  "labels_equal": bool((o.labels.cpu().numpy() == sk.labels_).all())})
        del x
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
