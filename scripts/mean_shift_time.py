"""Time mean_shift against the composition it replaces (one GPU, blobs data).

Workloads (n rows x d, seeding):
  1000000 x 32, bin seeding
  50000 x 128, every row a seed
  20000 x 300, every row a seed
Blobs around 16 centres (data()).
Arms:
  fused        mean_shift, the whole fit (CUDA events, after one warm-up fit); from the library's profiling events the
               time of every iteration (the first and the last one that had an active seed are printed); from a
               torch.profiler run of its own the summed time of ms_sum_kernel, against its MMA bound (2 s n 64 nkb flops
               per iteration at 989 TFLOP/s, the data sheet's dense fp16 rate)
  composition  the same iterations built from eps_neighbors_l2sq, adj.float() and a torch fp32 matmul of the active seeds
               against the rows, with the same stop rule; the centres from the final means by the contract's merge, order
               and walk (on the host), the labels by fused_l2_nn
The composition's centres and labels are compared with the fit's before any time is printed.  Prints the card and its
power limit, then one JSON line per workload.

  python scripts/mean_shift_time.py [--only 0,1,2]
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
import mean_shift_ref as R  # noqa: E402
from measure import card, time_ms  # noqa: E402
from raft_b200 import _lib  # noqa: E402
from raft_b200.cluster import mean_shift  # noqa: E402
from raft_b200.distance import fused_l2_nn_argmin  # noqa: E402
from raft_b200.neighbors.epsilon_neighborhood import eps_neighbors_l2sq  # noqa: E402

WORKLOADS = [(1000000, 32, True), (50000, 128, False), (20000, 300, False)]
H = 1.0


def data(n, d, bins, seed=5):
    """16 blobs.  For bin seeding the blobs sit on bin centres with 0.05 h of noise per coordinate, so their rows fall
    into a few bins; otherwise the rows lie about 0.7 h from their centre (about h from each other), so a seed first
    reaches part of its blob and climbs to its centre over a few iterations."""
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(16, d)) * (12.0 * H / np.sqrt(2))
    if bins:
        c = np.rint(c / H) * H
    x = c[rng.integers(0, 16, n)] + rng.normal(size=(n, d)) * (0.05 * H if bins else 0.7 * H / np.sqrt(d))
    return torch.from_numpy(x.astype(np.float32)).cuda()


def composed(x, seeds, max_iter=300):
    e = float(np.float32(H * H))
    means = seeds.clone()
    s = len(seeds)
    state = torch.zeros(s, dtype=torch.int32, device="cuda")
    iters = torch.zeros(s, dtype=torch.int64, device="cuda")
    inten = torch.zeros(s, dtype=torch.int64, device="cuda")
    for _ in range(max_iter + 1):
        act = torch.nonzero(state == 0).flatten()
        if len(act) == 0:
            break
        for a0 in range(0, len(act), 8192):
            idx = act[a0:a0 + 8192]
            adj, _ = eps_neighbors_l2sq(means[idx], x, e)
            A = torch.as_tensor(adj, device="cuda").float()
            cnt = A.sum(1)
            new = (A @ x) / cnt.clamp(min=1)[:, None]
            shift = (new.double() - means[idx].double()).norm(dim=1)
            drop = cnt == 0
            stop = ~drop & ((shift <= 1e-3 * H) | (iters[idx] == max_iter))
            go = ~drop & ~stop
            means[idx[~drop]] = new[~drop]
            inten[idx[~drop]] = cnt[~drop].long()
            state[idx[drop]] = 2
            state[idx[stop]] = 1
            iters[idx[go]] += 1
    keep = (state == 1).cpu().numpy()
    m = means.cpu().numpy()[keep]
    it = inten.cpu().numpy()[keep]
    cand = {}
    for row, c in zip(m, it):
        cand[row.tobytes()] = max(cand.get(row.tobytes(), 0), int(c))
    items = sorted(((c, np.frombuffer(k, np.float32)) for k, c in cand.items()),
                   key=lambda t: (t[0], tuple(R.ordered_bits(t[1]))), reverse=True)
    C = torch.from_numpy(np.stack([v for _, v in items])).cuda()
    W, _ = eps_neighbors_l2sq(C, C, e)
    W = torch.as_tensor(W, device="cuda")
    W = (W | W.T).cpu().numpy()
    sup = np.zeros(len(C), bool)
    kept = []
    for i in range(len(C)):
        if not sup[i]:
            kept.append(i)
            sup |= W[i]
    centres = C[kept]
    labels = torch.as_tensor(fused_l2_nn_argmin(x, centres, sqrt=False), device="cuda")
    return centres, labels, int(iters.max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    gpu = card()
    print("card: %s, power limit %s W" % (gpu["name"], gpu["power_limit"]), flush=True)
    L = _lib.lib()
    for wi in [int(s) for s in a.only.split(",") if s] or range(len(WORKLOADS)):
        n, d, bins = WORKLOADS[wi]
        x = data(n, d, bins)
        fit = lambda: mean_shift(x, bandwidth=H, bin_seeding=bins)   # noqa: E731
        _lib.check(L.b2d_profile_begin(512))
        res = fit()
        ms_it = torch.zeros(512, dtype=torch.float32)
        cnt = torch.zeros(1, dtype=torch.int32)
        _lib.check(L.b2d_profile_end(ms_it.data_ptr(), 512, cnt.data_ptr()))
        per_iter = ms_it[: int(cnt.item())].tolist()
        t_fit = time_ms(fit, 1, warmup=0)[0]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fit()
            torch.cuda.synchronize()
        sum_us = sum(e.device_time_total for e in prof.key_averages() if "ms_sum_kernel" in e.key)
        steps = res.n_iter + 1
        # seeds per iteration: every seed enters every iteration until the last one stops
        seeds = int(torch.from_numpy(R.bin_seeds(x.cpu().numpy(), H)).shape[0]) if bins else n
        mma_ms = 2.0 * seeds * n * 64 * ((d + 31) // 32) * steps / 989e12 * 1e3
        torch.cuda.synchronize()
        sd = torch.from_numpy(R.bin_seeds(x.cpu().numpy(), H)).cuda() if bins else x
        comp = composed(x, sd)
        t_comp = time_ms(lambda: composed(x, sd), 1, warmup=0)[0]
        same_labels = bool(torch.equal(comp[1].int(), res.labels))
        err = float((comp[0] - res.cluster_centers).abs().max()) if comp[0].shape == res.cluster_centers.shape else None
        print(json.dumps({"n": n, "d": d, "bin_seeding": bins, "seeds": seeds, "n_centers": len(res.cluster_centers),
                          "n_iter": res.n_iter, "fit_ms": round(t_fit, 3), "first_iter_ms": round(per_iter[0], 3),
                          "last_iter_ms": round(per_iter[res.n_iter], 3), "sum_kernel_ms": round(sum_us / 1e3, 3),
                          "sum_kernel_mma_bound_ms": round(mma_ms, 3), "composition_ms": round(t_comp, 3),
                          "composition_n_centers": len(comp[0]), "composition_n_iter": comp[2],
                          "same_labels": same_labels, "max_centre_diff": err, "card": gpu["name"],
                          "power_limit_w": gpu["power_limit"]}), flush=True)


if __name__ == "__main__":
    main()
