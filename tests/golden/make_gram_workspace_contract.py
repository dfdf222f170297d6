"""Generates tests/golden/gram_workspace_contract.json (run here, without a GPU; the output is committed).

The workspace contract of b2d_gram_matrix, in the format and with the conventions of make_workspace_contract.py:
  bytes   b2d_gram_matrix_workspace_bytes for every kernel id (and two invalid ones) and dtype over the shape grid of the
          b2d_eps_neighbors_l2sq_workspace_bytes entry;
  errors  (status, b2d_last_error()) of b2d_gram_matrix given a null workspace, one byte too few at an aligned address, or
          the full size at an odd address, for a few kernel x dtype x layout combinations, every other argument valid.
Pointers are fake addresses: a case that returns B2D_OK or B2D_ERR_CUDA got past validation and is refused.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from make_workspace_contract import BIG_M, D, DTYPES, KS, NEG, ODD, WS  # noqa: E402
from raft_b200 import _lib  # noqa: E402

OUT = os.path.join(HERE, "gram_workspace_contract.json")
KERNEL_IDS = list(range(-1, 5))   # LINEAR, POLYNOMIAL, RBF, TANH and one invalid id on either side


def byte_queries():
    edges = [(0, 29, 32), (37, 0, 32), (37, 29, 0)] + NEG
    shapes = [(37, 29, k) for k in KS] + edges + [(BIG_M, 1000, 96), (1000, 1 << 20, 128)]
    return {"b2d_gram_matrix_workspace_bytes": [(kr, dt) + s for kr in KERNEL_IDS for dt in DTYPES for s in shapes]}


def error_cases(L):
    """(name, function, arguments before the workspace pair, bytes needed, has an alignment check)"""
    gw = L.b2d_gram_matrix_workspace_bytes
    m, n, k = 300, 500, 96
    return [
        ("gram rbf f32", "b2d_gram_matrix", [None, 2, 0, 0.5, 0.0, 0, D, k, D, k, D, n, m, n, k, 1], gw(2, 0, m, n, k), True),
        ("gram polynomial f16 col-major", "b2d_gram_matrix", [None, 1, 3, 0.1, 1.0, 1, D, m, D, n, D, m, m, n, k, 0],
         gw(1, 1, n, m, k), True),
        ("gram tanh f32 k=400", "b2d_gram_matrix", [None, 3, 0, 0.1, -1.0, 0, D, 400, D, 400, D, n, m, n, 400, 1],
         gw(3, 0, m, n, 400), True),
        ("gram linear f64", "b2d_gram_matrix", [None, 0, 0, 1.0, 0.0, 2, D, k, D, k, D, n, m, n, k, 1], gw(0, 2, m, n, k), False),
        ("gram rbf f64 col-major", "b2d_gram_matrix", [None, 2, 0, 0.5, 0.0, 2, D, m, D, n, D, m, m, n, k, 0],
         gw(2, 2, n, m, k), False),
    ]


def main():
    L = _lib.lib()
    out = {"bytes": {}, "errors": []}
    for fn, cases in byte_queries().items():
        out["bytes"][fn] = [list(a) + [getattr(L, fn)(*a)] for a in cases]
    for name, fn, args, need, aligned in error_cases(L):
        assert 0 < need < 2 ** 63, (name, need)
        variants = [("null", None, need), ("short", WS, need - 1)] + ([("odd", ODD, need)] if aligned else [])
        for case, ws, nbytes in variants:
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
