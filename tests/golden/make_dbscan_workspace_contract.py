"""Generates tests/golden/dbscan_workspace_contract.json (run here, without a GPU; the output is committed): the
workspace contract of b2d_dbscan_workspace_bytes / b2d_dbscan_fit in the format of make_workspace_contract.py, whose
recorder and writer it uses.
  bytes   row counts around the 16-column adjacency pitch and the 256-column batch step, every k of the other fixtures,
          and batch sizes from the 2^30 default (0) through the 256-column floor (1) to one batch of every column;
  errors  a null, short or misaligned workspace for the euclidean, cosine (batched, optional outputs null) and
          sqeuclidean (NaN eps) fits."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_workspace_contract as wc  # noqa: E402

DB_MS = [1, 15, 16, 256, 257, 32768, 100000, 1000000]
DB_BATCH = [0, 1, 1 << 20, 1 << 26, (1 << 30) + 1, 1 << 40]


def dbscan_byte_queries():
    q = [(m, d, b) for m in DB_MS for d in wc.KS for b in DB_BATCH] + \
        [(0, 32, 0), (-1, 32, 0), (37, -1, 0), (37, 32, -1)]
    return {"b2d_dbscan_workspace_bytes": q}


def dbscan_error_cases(L):
    m, d, D = 5000, 96, wc.D
    return [
        ("dbscan euclidean", "b2d_dbscan_fit", [None, 1, D, d, m, d, 0.5, 5, 0, D, D, D],
         L.b2d_dbscan_workspace_bytes(m, d, 0), True),
        ("dbscan cosine batched", "b2d_dbscan_fit", [None, 2, D, d + 3, m, d, 0.1, 1, 1 << 20, D, None, None],
         L.b2d_dbscan_workspace_bytes(m, d, 1 << 20), True),
        ("dbscan sqeuclidean NaN eps", "b2d_dbscan_fit", [None, 0, D, d, m, d, float("nan"), 50, 12345, D, D, None],
         L.b2d_dbscan_workspace_bytes(m, d, 12345), True),
    ]


if __name__ == "__main__":
    # the shared writer over this one fixture
    wc.FIXTURES = {"dbscan_workspace_contract.json": (dbscan_byte_queries, dbscan_error_cases)}
    wc.main()
