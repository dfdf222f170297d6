"""Time the k-means fit (raft_b200.cluster.kmeans) against the composition a user would write without it:
fused_l2_nn_argmin + a torch index_add_ mean per iteration, with a host convergence test.  Blobs of 1 000 000 x 128,
Array init, tol = 0, max_iter = 20.  Prints one JSON line per measurement, and writes them to --out."""
import argparse
import json
import os
import sys
from statistics import median

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import kmeans_ref  # noqa: E402
from measure import card, time_ms  # noqa: E402
from raft_b200 import _lib  # noqa: E402
from raft_b200.cluster import KMeansParams, fit, init_plus_plus  # noqa: E402
from raft_b200.common import DeviceResources  # noqa: E402
from raft_b200.distance import fused_l2_nn  # noqa: E402


def composition(x, x64, c0, iters, tol, h):
    # x64: x in fp64, converted once by the caller, so the loop holds only the per-iteration work
    c = c0.clone()
    m, k = x.shape
    nc = c.shape[0]
    ones = torch.ones(m, dtype=torch.float64, device="cuda")
    for it in range(iters):
        lab, _ = fused_l2_nn(x, c, sqrt=False, handle=h)
        s = torch.zeros((nc, k), dtype=torch.float64, device="cuda").index_add_(0, lab.long(), x64)
        n = torch.zeros(nc, dtype=torch.float64, device="cuda").index_add_(0, lab.long(), ones)
        new = torch.where(n[:, None] > 0, s / n.clamp(min=1)[:, None], c.double()).float()
        shift = float(((new.double() - c.double()) ** 2).sum())   # host convergence test
        c = new
        if shift < tol:
            break
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=1000000)
    ap.add_argument("--k", type=int, default=128)
    ap.add_argument("--clusters", default="16,256,4096")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = [{"gpu": card()}]
    print(json.dumps(rows[0]), flush=True)
    h = DeviceResources()
    for nc in [int(v) for v in a.clusters.split(",")]:
        x_np, _, _ = kmeans_ref.blobs(a.m, a.k, nc, seed=nc, spread=0.3)
        x = torch.from_numpy(x_np).cuda()
        c0 = x[torch.from_numpy(np.random.default_rng(nc).choice(a.m, nc, replace=False)).cuda()].contiguous()
        cf = torch.empty_like(c0)

        def run_fit(max_iter=a.iters, tol=0.0):
            cf.copy_(c0)
            return fit(KMeansParams(n_clusters=nc, max_iter=max_iter, tol=tol, init_method="Array"), x, cf, handle=h)

        # a call whose result is used is its own warm-up
        out = run_fit()
        t_fit = median(time_ms(run_fit, a.reps, warmup=0))
        fused_c = cf.clone()
        _lib.check(_lib.lib().b2d_set_option(b"nn_screen", 0))
        x64 = x.double()
        comp_c = composition(x, x64, c0, a.iters, 0.0, h)
        t_comp = median(time_ms(lambda: composition(x, x64, c0, a.iters, 0.0, h), a.reps, warmup=0))
        del x64
        _lib.check(_lib.lib().b2d_set_option(b"nn_screen", 1))
        lab_f, _ = fused_l2_nn(x, fused_c, sqrt=False, handle=h)
        lab_c, _ = fused_l2_nn(x, comp_c, sqrt=False, handle=h)
        ia = fused_c.view(torch.int32).long()
        ib = comp_c.view(torch.int32).long()
        # default tol: the no-op iterations after convergence
        conv = run_fit(300, 1e-4)
        t300 = median(time_ms(lambda: run_fit(300, 1e-4), a.reps, warmup=0))
        tn = median(time_ms(lambda: run_fit(conv.n_iter, 1e-4), a.reps))
        byte_floor_ms = 8.0 * a.m * a.k / 3.35e12 * 1e3
        r = {"n_clusters": nc, "m": a.m, "k": a.k, "fit_ms_per_iter": t_fit / out.n_iter,
             "composition_ms_per_iter": t_comp / a.iters, "byte_floor_ms_per_iter": byte_floor_ms,
             "tensor_floor_ms_per_iter": 3 * 2.0 * a.m * nc * a.k / 989e12 * 1e3,
             "noop_iters": 300 - conv.n_iter, "noop_ms_total": t300 - tn, "n_iter_default_tol": conv.n_iter,
             "labels_equal": bool((lab_f == lab_c).all()), "max_centroid_ulps": int((ia - ib).abs().max())}
        rows.append(r)
        print(json.dumps(r), flush=True)
    x_np, _, _ = kmeans_ref.blobs(a.m, a.k, 1024, seed=1, spread=0.3)
    x = torch.from_numpy(x_np).cuda()
    t_pp = time_ms(lambda: init_plus_plus(x, n_clusters=1024, seed=0, handle=h), 1)[0]
    rows.append({"kmeans_plus_plus_ms": t_pp, "n_clusters": 1024, "m": a.m, "k": a.k})
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
