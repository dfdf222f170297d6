"""Time kernel_density against the composition it replaces (one GPU, blobs data, unit weights).

Workloads (m queries x n dataset rows x d), for the gaussian and the epanechnikov kernel:
  100000 x 100000 x 128
  1000000 x 100000 x 32
Arms, run alternately (fused, composition, fused, ...), median of --runs each (CUDA events after one warm-up call each):
  fused        kernel_density, the whole call; from the library's profiling events the EPI_KDE tensor kernels alone
               (summed over the slabs), and the rest of the call (operand preparation, weights, fold, finish)
  composition  pairwise_distance(sqeuclidean) in query slabs of at most 1 GiB, then per row torch.logsumexp of
               -d 0.5 / h^2 (gaussian) or the log of the sum of max(1 - d / h^2, 0) over d < h^2 (epanechnikov), plus
               the normalisation
The bandwidth puts about 1000 dataset rows inside h per query on average (from the distances of 64 queries).  Before any
time is printed, the largest |fused - composition| over all rows is computed and reported.  Prints the card and its
power limit, then one JSON line per (workload, kernel).

  python scripts/kde_time.py [--runs 3] [--only 0,1]
"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import kde_ref  # noqa: E402
import oracle  # noqa: E402
from measure import card, time_ms  # noqa: E402
from raft_b200 import _lib  # noqa: E402
from raft_b200.common import DeviceResources  # noqa: E402
from raft_b200.distance import pairwise_distance  # noqa: E402
from raft_b200.neighbors import kernel_density  # noqa: E402

WORKLOADS = [(100000, 100000, 128), (1000000, 100000, 32)]
KERNELS = ["gaussian", "epanechnikov"]
SLAB_BYTES = 1 << 30   # dense slab of the composition


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    gpu = card()
    pl = "%s W, %s MHz" % (gpu["power_limit"], gpu["clocks_max_sm"])
    print("card: %s, power limit, max SM clock: %s" % (gpu["name"], pl), flush=True)
    hd = DeviceResources()
    L = _lib.lib()
    sel = [int(s) for s in a.only.split(",") if s] or range(len(WORKLOADS))
    for wi in sel:
        m, n, d = WORKLOADS[wi]
        c = oracle.make_blobs(16, d, seed=7)[2]
        q = torch.from_numpy(oracle.make_blobs(m, d, seed=11, centers=c)[0]).cuda()
        x = torch.from_numpy(oracle.make_blobs(n, d, seed=13, centers=c)[0]).cuda()
        slab = max(1, min(m, SLAB_BYTES // (4 * n)))
        dist = torch.empty((slab, n), dtype=torch.float32, device="cuda")
        pairwise_distance(q[:64], x, out=dist[:64], metric="sqeuclidean", handle=hd)
        hd.sync()
        h = math.sqrt(float(torch.kthvalue(dist[:64].flatten(), 1000 * 64).values))   # ~1000 rows within h per query
        for kernel in KERNELS:
            ln = kde_ref.log_norm(kernel, h, d) - math.log(n)
            h2 = kde_ref.h2_of(h)

            def fused():
                return kernel_density(x, q, bandwidth=h, kernel=kernel, handle=hd)

            def composition():
                out = torch.empty(m, dtype=torch.float64, device="cuda")
                with torch.cuda.stream(hd.torch_stream):
                    for r0 in range(0, m, slab):
                        s = min(slab, m - r0)
                        dd = dist[:s]
                        pairwise_distance(q[r0:r0 + s], x, out=dd, metric="sqeuclidean", handle=hd)
                        if kernel == "gaussian":
                            r = torch.logsumexp(dd * (-0.5 / (h * h)), dim=1)
                        else:
                            r = torch.where(dd < h2, (1.0 - dd * (1.0 / (h * h))).clamp_min(0.0), 0.0).sum(1).log()
                        out[r0:r0 + s] = r.double() + ln
                return out

            got = fused()
            want = composition()
            hd.sync()
            fin = torch.isfinite(want) & torch.isfinite(got)
            max_abs = float((got - want)[fin].abs().max())
            same_inf = bool(torch.equal(torch.isfinite(got), torch.isfinite(want)))
            del want
            ts = {"fused": [], "composition": []}
            for _ in range(a.runs):
                for arm, fn in (("fused", fused), ("composition", composition)):
                    ts[arm] += time_ms(lambda: (fn(), hd.sync()), 1, warmup=0)
            kern = []
            ws = torch.empty(L.b2d_kde_workspace_bytes(m, n, d, 0), dtype=torch.uint8, device="cuda")
            for _ in range(a.runs):
                _lib.check(L.b2d_profile_begin(64))
                _lib.check(L.b2d_kde_score_samples(hd.stream_ptr, ["gaussian", "tophat", "epanechnikov"].index(kernel),
                                                   h, x.data_ptr(), d, None, q.data_ptr(), d, m, n, d, 0, got.data_ptr(),
                                                   ws.data_ptr(), ws.numel()))
                ms = torch.zeros(64, dtype=torch.float32)
                cnt = torch.zeros(1, dtype=torch.int32)
                _lib.check(L.b2d_profile_end(ms.data_ptr(), 64, cnt.data_ptr()))
                kern.append(float(ms[:int(cnt)].sum()))
            del ws
            fm, cm, km = statistics.median(ts["fused"]), statistics.median(ts["composition"]), statistics.median(kern)
            print(json.dumps({"m": m, "n": n, "d": d, "kernel": kernel, "bandwidth": round(h, 4),
                              "card": gpu["name"], "power_limit_max_sm_clock": pl,
                              "fused_ms": round(fm, 3), "composition_ms": round(cm, 3), "speedup": round(cm / fm, 2),
                              "fused_kernel_ms": round(km, 3), "fused_rest_ms": round(fm - km, 3),
                              "max_abs_diff": max_abs, "same_finite_rows": same_inf,
                              "runs": {k: [round(t, 3) for t in v] for k, v in ts.items()}}), flush=True)
        del q, x, dist
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
