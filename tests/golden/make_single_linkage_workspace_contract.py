"""Generates tests/golden/single_linkage_workspace_contract.json (run here, without a GPU; the output is committed).

The workspace contract of the single-linkage entry points, in the format and with the conventions of
make_workspace_contract.py:
  bytes   b2d_single_linkage_workspace_bytes(m, d, c) over row counts from 1 to 10^6 (around the 2048-row sort blocks and
          the 2^20-row tile-class cap), the d of the other queries, c from -5 to 60 (n_nb from 2 to past 64), and
          negative extents; b2d_mst_workspace_bytes(n_vertices, n_edges) over a grid and negative extents;
  errors  (status, b2d_last_error()) of b2d_single_linkage and b2d_mst given a null workspace, one byte too few at an
          aligned address, or the full size at an odd address, every other argument valid.
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

OUT = os.path.join(HERE, "single_linkage_workspace_contract.json")
MS = [1, 2, 37, 2048, 2049, 100000, (1 << 20) + 1, 1000000]
CS = [-5, 1, 15, 45, 60]
NS = [0, 1, 1000, 1000000]
ES = [0, 5000, 10 ** 7]


def byte_queries():
    sl = [(m, d, c) for m in MS for d in KS for c in CS] + [(0, 32, 15), (-1, 32, 15), (37, -1, 15)]
    mst = [(n, e) for n in NS for e in ES] + [(-1, 10), (10, -1)]
    return {"b2d_single_linkage_workspace_bytes": sl, "b2d_mst_workspace_bytes": mst}


def error_cases(L):
    """(name, function, arguments before the workspace pair, bytes needed)"""
    m, d, n, e = 5000, 96, 3000, 20000
    return [
        ("single_linkage euclidean", "b2d_single_linkage", [None, 1, D, d, m, d, 15, 7, D, D, D, D, D],
         L.b2d_single_linkage_workspace_bytes(m, d, 15)),
        ("single_linkage sqeuclidean c=40", "b2d_single_linkage", [None, 0, D, d + 3, m, d, 40, 1, D, D, D, D, D],
         L.b2d_single_linkage_workspace_bytes(m, d, 40)),
        ("mst", "b2d_mst", [None, D, D, D, n, e, D, D, D, D, D], L.b2d_mst_workspace_bytes(n, e)),
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
