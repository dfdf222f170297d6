"""Generates tests/golden/kmeans_balanced_workspace_contract.json (run without a GPU; the output is committed), in the
format and with the recorder of make_workspace_contract.py:
  bytes   b2d_kmeans_balanced_workspace_bytes over the k-means row counts, every k of the other fixtures, cluster counts
          from 1 to 65536 (G = 1 to 256 mesoclusters), and the queries that return SIZE_MAX (negative extents);
  errors  b2d_kmeans_balanced_fit with and without its optional outputs, given a null, short or misaligned workspace.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_workspace_contract as mwc  # noqa: E402

KB_MS = [1, 100, 2047, 2048, 100000, 10 ** 6]
KB_NCS = [1, 2, 3, 17, 1000, 65536]


def balanced_byte_queries():
    q = [(m, k, nc) for m in KB_MS for k in mwc.KS for nc in KB_NCS if nc <= m] + \
        [(0, 32, 0), (37, 0, 4), (-1, 32, 4), (37, -1, 4), (37, 32, -1)]
    return {"b2d_kmeans_balanced_workspace_bytes": q}


def balanced_error_cases(L):
    wb = L.b2d_kmeans_balanced_workspace_bytes
    D = mwc.D
    m, k, nc = 5000, 96, 40
    return [
        ("balanced_fit", "b2d_kmeans_balanced_fit", [None, nc, 20, 3, D, k, m, k, D, None, None], wb(m, k, nc), True),
        ("balanced_fit with labels and sizes", "b2d_kmeans_balanced_fit", [None, nc, 5, 3, D, k, m, k, D, D, D],
         wb(m, k, nc), True),
    ]


def main():
    L = mwc._lib.lib()
    out = mwc.record(L, balanced_byte_queries, balanced_error_cases)
    path = os.path.join(HERE, "kmeans_balanced_workspace_contract.json")
    with open(path, "w") as fh:   # one case per line, as the other fixtures
        fh.write('{"bytes": {\n')
        fh.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                            for fn, rows in out["bytes"].items()))
        fh.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
