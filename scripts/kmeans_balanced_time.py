"""Times raft_b200.cluster.kmeans_balanced.fit_predict on blobs and compares it with a k-means||-seeded kmeans.fit of the
same iteration budget: fit time (CUDA events, median of --reps), its split by stage, inertia ratio and cluster-size
spreads.  The stages are the measured regions the library records between b2d_profile_begin and b2d_profile_end: in
launch order stage 0 (mesoclusters), stage 1 (allocation, gather, tables and the fine EM), stage 1's n_iters masked
arg-min launches, stage 2 (the final pass).  Prints one
JSON line per measurement (with the card name and its power limit); writes them to a file only with --out."""
import argparse
import ctypes
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from measure import card, time_ms  # noqa: E402
from raft_b200.cluster import KMeansParams, fit as km_fit, predict as km_predict  # noqa: E402
from raft_b200 import _lib  # noqa: E402
from raft_b200.cluster import kmeans_balanced as kb  # noqa: E402


def stage_ms(fn, n_iters):
    """(stage 0, stage 1, stage 1's masked arg-min launches summed, stage 2) in ms for one call of fn."""
    L = _lib.lib()
    torch.cuda.synchronize()
    _lib.check(L.b2d_profile_begin(64 + n_iters))
    fn()
    buf = (ctypes.c_float * (64 + n_iters))()
    cnt = ctypes.c_int(0)
    _lib.check(L.b2d_profile_end(buf, 64 + n_iters, ctypes.byref(cnt)))
    ms = list(buf)[:cnt.value]
    assert cnt.value == 3 + n_iters, cnt.value
    return ms[0], ms[1], sum(ms[2:2 + n_iters]), ms[2 + n_iters]


def blobs(m, k, centers, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.rand((centers, k), generator=g, device="cuda") * 20 - 10
    lab = torch.randint(0, centers, (m,), generator=g, device="cuda")
    return (c[lab] + torch.randn((m, k), generator=g, device="cuda") * 1.5).contiguous()


def spreads(sizes):
    s = sizes.double()
    return float(s.min() / s.mean()), float(s.max() / s.mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1000000)
    ap.add_argument("--k", type=int, default=128)
    ap.add_argument("--clusters", type=int, nargs="+", default=[1024, 16384, 65536])
    ap.add_argument("--n-iters", type=int, default=20)
    ap.add_argument("--kmeans-max", type=int, default=4096, help="largest n_clusters for the kmeans.fit comparison")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = card()
    x = blobs(a.m, a.k, 2048, 0)
    lines = []
    for nc in a.clusters:
        p = kb.KMeansBalancedParams(n_iters=a.n_iters)
        c, lab, sizes = kb.fit_predict(p, x, nc)   # the warm-up; every fit returns the same result
        ms = statistics.median(time_ms(lambda: kb.fit_predict(p, x, nc), a.reps, warmup=0))
        c = torch.as_tensor(c, device="cuda")
        _, inertia = km_predict(KMeansParams(n_clusters=nc), x, c)
        lo, hi = spreads(torch.as_tensor(sizes, device="cuda"))
        s0, s1, s1_argmin, s2 = stage_ms(lambda: kb.fit_predict(p, x, nc), a.n_iters)
        rec = dict(what="kmeans_balanced.fit_predict", m=a.m, k=a.k, n_clusters=nc, n_iters=a.n_iters, ms=ms,
                   inertia=inertia, stage0_ms=s0, stage1_ms=s1,
                   stage1_masked_argmin_ms=s1_argmin, stage2_ms=s2, min_over_avg=lo, max_over_avg=hi, gpu=gpu["name"],
                   power_limit=gpu["power_limit"])
        if nc <= a.kmeans_max:
            iters = a.n_iters * 2 + max(a.n_iters // 10, 2)
            kp = KMeansParams(n_clusters=nc, max_iter=iters, tol=0.0, oversampling_factor=2.0)
            o = km_fit(kp, x)   # the warm-up; seeded, so every fit returns the same result
            kms = time_ms(lambda: km_fit(kp, x), 1, warmup=0)[0]
            klab, _ = km_predict(KMeansParams(n_clusters=nc), x, o.centroids)
            klo, khi = spreads(torch.bincount(torch.as_tensor(klab, device="cuda").long(), minlength=nc))
            rec.update(kmeans_ms=kms, kmeans_max_iter=iters, inertia_over_kmeans=inertia / o.inertia,
                       kmeans_min_over_avg=klo, kmeans_max_over_avg=khi)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
