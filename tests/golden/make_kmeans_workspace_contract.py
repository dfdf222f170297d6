"""Generates tests/golden/kmeans_workspace_contract.json (run here, without a GPU; the output is committed).

The workspace contract of the k-means entry points, in the format and with the conventions of make_workspace_contract.py:
  bytes   b2d_kmeans_workspace_bytes(m, k, n_clusters) over a grid of row counts (including ones past the histogram
          cap), the k of the other queries, cluster counts from 1 to 10^5, and negative extents;
  errors  (status, b2d_last_error()) of b2d_kmeans_fit / predict / update_centroids / init_plus_plus given a null
          workspace, one byte too few at an aligned address, or the full size at an odd address, every other argument
          valid.
Pointers are fake addresses: a case that returns B2D_OK or B2D_ERR_CUDA got past validation and is refused.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from make_workspace_contract import D, KS, ODD, WS  # noqa: E402
from raft_b200 import _lib  # noqa: E402

OUT = os.path.join(HERE, "kmeans_workspace_contract.json")
MS = [1, 37, 2048, 2049, 100000, 1000000]
NCS = [1, 17, 1000, 100000]
NEG = [(-1, 32, 4), (37, -1, 4), (37, 32, -1)]


def byte_queries():
    shapes = [(m, k, nc) for m in MS for k in KS for nc in NCS] + [(0, 32, 0), (37, 0, 4)] + NEG
    return {"b2d_kmeans_workspace_bytes": shapes}


def error_cases(L):
    """(name, function, arguments before the workspace pair, bytes needed)"""
    wb = L.b2d_kmeans_workspace_bytes
    m, k, nc = 5000, 96, 40
    return [
        ("fit array", "b2d_kmeans_fit", [None, nc, 20, 1e-4, 2, 1, 0, 0, D, k, None, m, k, D, D, D], wb(m, k, nc)),
        ("fit k-means++ weighted n_init=3", "b2d_kmeans_fit", [None, nc, 20, 1e-4, 0, 3, 7, 1, D, k, D, m, k, D, D, D],
         wb(m, k, nc)),
        ("predict", "b2d_kmeans_predict", [None, D, k, None, m, k, D, nc, D, D, 1], wb(m, k, nc)),
        ("update_centroids", "b2d_kmeans_update_centroids", [None, D, k, D, D, m, k, D, nc, D, None], wb(m, k, nc)),
        ("init_plus_plus", "b2d_kmeans_init_plus_plus", [None, D, k, None, m, k, nc, 3, D], wb(m, k, nc)),
    ]


def main():
    L = _lib.lib()
    out = {"bytes": {}, "errors": []}
    for fn, cases in byte_queries().items():
        out["bytes"][fn] = [list(a) + [getattr(L, fn)(*a)] for a in cases]
    for name, fn, args, need in error_cases(L):
        assert 0 < need < 2 ** 63, (name, need)
        for case, ws, nbytes in [("null", None, need), ("short", WS, need - 1), ("odd", ODD, need)]:
            a = args + [ws, nbytes]
            rc = getattr(L, fn)(*a)
            if rc in (_lib.B2D_OK, _lib.B2D_ERR_CUDA):
                raise SystemExit(f"{name} / {case}: status {rc} -- the call got past validation; not recorded")
            out["errors"].append({"name": name, "case": case, "fn": fn, "args": a, "rc": rc,
                                  "msg": L.b2d_last_error().decode()})
    with open(OUT, "w") as f:   # one case per line, as in workspace_contract.json
        f.write('{"bytes": {\n')
        f.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                           for fn, rows in out["bytes"].items()))
        f.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", OUT, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
