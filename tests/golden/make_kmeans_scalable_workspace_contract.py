"""Generates tests/golden/kmeans_scalable_workspace_contract.json (run without a GPU; the output is committed), in the
format and with the recorder of make_workspace_contract.py:
  bytes   b2d_kmeans_scalable_workspace_bytes over the k-means row counts and cluster counts, every k of the other
          fixtures, oversampling factors from 0.01 (the (n_clusters - 1) / 8 floor) to 10^6 (L clamped to m), and the
          queries that return SIZE_MAX: negative extents, a factor that is 0, negative, NaN or infinite, and a candidate
          set of 2^31 rows or more;
  errors  init_scalable and fit_scalable (weighted, n_init = 3) given a null, short or misaligned workspace.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_workspace_contract as mwc  # noqa: E402

KS_MS = [1, 100, 2047, 2048, 100000, 10 ** 6]
KS_NCS = [1, 17, 1000]
KS_FS = [0.01, 0.5, 2.0, 1e6]


def scalable_byte_queries():
    q = [(m, k, nc, f) for m in KS_MS for k in mwc.KS for nc in KS_NCS if nc <= m for f in KS_FS] + \
        [(0, 32, 0, 2.0), (37, 0, 4, 2.0), (-1, 32, 4, 2.0), (37, -1, 4, 2.0), (37, 32, -1, 2.0),
         (37, 32, 4, 0.0), (37, 32, 4, -1.0), (37, 32, 4, float("nan")), (37, 32, 4, float("inf")),
         (1 << 30, 8, 1 << 28, 1.0), (1 << 30, 8, 1 << 28, 0.5), ((1 << 31) - 1, 8, 1, 1e9)]
    return {"b2d_kmeans_scalable_workspace_bytes": q}


def scalable_error_cases(L):
    wb = L.b2d_kmeans_scalable_workspace_bytes
    D = mwc.D
    m, k, nc, f = 5000, 96, 40, 2.0
    return [
        ("init_scalable", "b2d_kmeans_init_scalable", [None, D, k, None, m, k, nc, f, 3, D, None, None], wb(m, k, nc, f),
         True),
        ("init_scalable weighted with candidates", "b2d_kmeans_init_scalable", [None, D, k, D, m, k, nc, 0.5, 3, D, D, D],
         wb(m, k, nc, 0.5), True),
        ("fit_scalable weighted n_init=3", "b2d_kmeans_fit_scalable",
         [None, nc, 20, 1e-4, f, 3, 7, 1, D, k, D, m, k, D, D, D], wb(m, k, nc, f), True),
    ]


def main():
    L = mwc._lib.lib()
    out = mwc.record(L, scalable_byte_queries, scalable_error_cases)
    path = os.path.join(HERE, "kmeans_scalable_workspace_contract.json")
    with open(path, "w") as fh:   # one case per line, as the other fixtures
        fh.write('{"bytes": {\n')
        fh.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                            for fn, rows in out["bytes"].items()))
        fh.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
