"""Time radius_neighbors against the compositions it replaces (one GPU, metric sqeuclidean).

Workloads (m queries x n dataset rows x k, blobs data), each at two radii: the squared distances that give about 100 and
about 1000 neighbours per query row (from a sample of the distances):
  100000 x 100000 x 128
  200000 x 1000000 x 32
Arms:
  fused        radius_neighbors, the whole call (count, the host read of nnz, fill), and its parts through the C ABI:
               count (prep, count kernel, scan), fill (prep, fill kernel, segmented sort, split) and, from the library's
               profiling events, the two tensor kernels alone; fill_prep_sort_split = fill - fill kernel
  pairwise     slabs of pairwise_distance, then <=, torch.nonzero, a gather and a per-row sort by the packed
               (distance, index) key: the same CSR, bit for bit
  eps          slabs of eps_neighbors_l2sq with torch.nonzero, the squared distances computed again from the norms and
               an inner product, and the same per-row sort (sqeuclidean only; its distances are not pairwise_distance's)
Before any time is printed, the fused CSR is checked equal to the pairwise composition's (indptr, indices, distance
bits) and the eps composition's rows are checked to hold the same columns.  Median of --runs calls per arm (CUDA events,
one warm-up call each).  Prints the card and its power limit, then one JSON line per (workload, radius).

  python scripts/radius_neighbors_time.py [--runs 3] [--only 0,1]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from measure import card, time_ms  # noqa: E402
from raft_b200 import _lib  # noqa: E402
from raft_b200.common import DeviceResources  # noqa: E402
from raft_b200.distance import pairwise_distance  # noqa: E402
from raft_b200.neighbors import eps_neighbors_l2sq, radius_neighbors  # noqa: E402

WORKLOADS = [(100000, 100000, 128), (200000, 1000000, 32)]
NEIGHBOURS = [100, 1000]
SLAB_BYTES = 4 << 30   # dense slab of the compositions


def packed_key(d, j):
    """oracle.pack_minloc in torch: ordered float bits << 32 | index"""
    b = d.view(torch.int32).to(torch.int64)
    b = torch.where(b < 0, b ^ 0x7FFFFFFF, b)
    return (b << 32) | (j & 0xFFFFFFFF)


def csr_of(rows, cols, vals, m):
    """CSR of the pairs (rows ascending, any column order), each row sorted by the packed key"""
    order = torch.sort(packed_key(vals, cols), stable=True).indices
    order = order[torch.sort(rows[order], stable=True).indices]
    indptr = torch.zeros(m + 1, dtype=torch.int64, device=rows.device)
    indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=m), 0)
    return indptr, cols[order], vals[order]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    gpu = card()
    pl = "%s W, %s MHz" % (gpu["power_limit"], gpu["clocks_max_sm"])
    print("card: %s, power limit, max SM clock: %s" % (gpu["name"], pl), flush=True)
    h = DeviceResources()
    L = _lib.lib()
    sel = [int(s) for s in a.only.split(",") if s] or range(len(WORKLOADS))
    for wi in sel:
        m, n, k = WORKLOADS[wi]
        c = oracle.make_blobs(16, k, seed=7)[2]
        q = torch.from_numpy(oracle.make_blobs(m, k, seed=11, centers=c)[0]).cuda()
        x = torch.from_numpy(oracle.make_blobs(n, k, seed=13, centers=c)[0]).cuda()
        slab = max(128, SLAB_BYTES // (4 * n) // 128 * 128)
        dist = torch.empty((slab, n), dtype=torch.float32, device="cuda")
        adj = torch.empty((slab, n), dtype=torch.bool, device="cuda")
        vd = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        pairwise_distance(q[:256], x, out=dist[:256], metric="sqeuclidean", handle=h)
        h.sync()
        sample = dist[:256].flatten()
        qn, xn = (q * q).sum(1), (x * x).sum(1)
        for nb in NEIGHBOURS:
            r = float(sample.kthvalue(max(1, int(nb / n * sample.numel()))).values)

            def fused():
                return radius_neighbors(x, q, r, metric="sqeuclidean", handle=h)

            def comp_pairwise():
                parts = []
                with torch.cuda.stream(h.torch_stream):
                    for r0 in range(0, m, slab):
                        s = min(slab, m - r0)
                        pairwise_distance(q[r0:r0 + s], x, out=dist[:s], metric="sqeuclidean", handle=h)
                        i, j = torch.nonzero(dist[:s] <= r, as_tuple=True)
                        parts.append((i + r0, j, dist[:s][i, j]))
                    return csr_of(*(torch.cat(t) for t in zip(*parts)), m)

            def comp_eps():
                parts = []
                with torch.cuda.stream(h.torch_stream):
                    for r0 in range(0, m, slab):
                        s = min(slab, m - r0)
                        eps_neighbors_l2sq(q[r0:r0 + s], x, r, adj=adj[:s], vd=vd, handle=h)
                        i, j = torch.nonzero(adj[:s], as_tuple=True)
                        qi = q[r0:r0 + s][i]
                        d = torch.clamp_min(qn[r0 + i] + xn[j] - 2.0 * (qi * x[j]).sum(1), 0.0)
                        parts.append((i + r0, j, d))
                    return csr_of(*(torch.cat(t) for t in zip(*parts)), m)

            got = fused()
            h.sync()
            want = comp_pairwise()
            h.sync()
            assert torch.equal(got[0], want[0]), "indptr differs from the pairwise composition"
            assert torch.equal(got[1], want[1]), "indices differ from the pairwise composition"
            assert torch.equal(got[2].view(torch.int32), want[2].view(torch.int32)), "distances differ"
            nnz = int(got[0][m])
            del want
            e = comp_eps()
            h.sync()
            assert torch.equal(e[0], got[0]), "eps composition: row degrees differ"
            rows = torch.repeat_interleave(torch.arange(m, device="cuda"), torch.diff(got[0]))
            assert torch.equal(torch.sort(rows * n + e[1]).values, torch.sort(rows * n + got[1]).values), \
                "eps composition: the rows hold other columns"
            del e, rows

            # the parts, through the C ABI with the library's profiling events around the tensor kernels
            indptr, indices, distances = got
            ws = torch.empty(L.b2d_radius_neighbors_workspace_bytes(m, n, k, nnz), dtype=torch.uint8, device="cuda")
            sp = h.stream_ptr

            def count():
                _lib.check(L.b2d_radius_neighbors_count(sp, indptr.data_ptr(), 0, q.data_ptr(), k, x.data_ptr(), k, m, n,
                                                        k, r, ws.data_ptr(), ws.numel()))

            def fill():
                _lib.check(L.b2d_radius_neighbors_fill(sp, indptr.data_ptr(), nnz, indices.data_ptr(),
                                                       distances.data_ptr(), 0, q.data_ptr(), k, x.data_ptr(), k, m, n, k,
                                                       r, ws.data_ptr(), ws.numel()))

            res = {}
            for arm, fn in (("fused_total", fused), ("count_call", count), ("fill_call", fill),
                            ("pairwise_composition", comp_pairwise), ("eps_composition", comp_eps)):
                ts = time_ms(lambda: (fn(), h.sync()), a.runs)
                res[arm] = {"median_ms": round(statistics.median(ts), 3), "ms": [round(t, 3) for t in ts]}
            kern = {}
            for arm, fn in (("count_kernel", count), ("fill_kernel", fill)):
                vals = []
                for _ in range(a.runs):
                    _lib.check(L.b2d_profile_begin(8))
                    fn()
                    ms = torch.zeros(8, dtype=torch.float32)
                    cnt = torch.zeros(1, dtype=torch.int32)
                    _lib.check(L.b2d_profile_end(ms.data_ptr(), 8, cnt.data_ptr()))
                    vals.append(float(ms[:int(cnt)].sum()))
                kern[arm] = round(statistics.median(vals), 3)
            res.update(kern)
            res["fill_prep_sort_split_ms"] = round(res["fill_call"]["median_ms"] - kern["fill_kernel"], 3)
            print(json.dumps({"m": m, "n": n, "k": k, "radius": r, "neighbours_per_row": round(nnz / m, 1), "nnz": nnz,
                              "card": gpu["name"], "power_limit_max_sm_clock": pl, **res}), flush=True)
            del ws
        del q, x, dist, adj, vd
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
