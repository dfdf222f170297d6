"""Generates tests/golden/radius_neighbors_workspace_contract.json (run without a GPU; the output is committed), in the format
and with the recorder of make_workspace_contract.py:
  bytes   b2d_radius_neighbors_workspace_bytes over row counts around the 64-row scan bound and the 1024-byte regions, every
          k of the other fixtures, and nnz from 0 (the count call) to 2^31 - 1, plus negative arguments;
  errors  the count and fill calls of every metric given a null, short or misaligned workspace.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_workspace_contract as mwc  # noqa: E402

RN_MS = [0, 1, 63, 64, 65, 255, 256, 100000, (1 << 31) - 1]
RN_NS = [1, 100000]
RN_NNZ = [0, 1, 1000, 10 ** 7, (1 << 31) - 1]


def radius_byte_queries():
    q = [(m, n, k, z) for m in RN_MS for n in RN_NS for k in mwc.KS for z in RN_NNZ] + \
        [(0, 0, 0, 0), (-1, 5, 8, 0), (5, -1, 8, 0), (5, 5, -1, 0), (5, 5, 8, -1)]
    return {"b2d_radius_neighbors_workspace_bytes": q}


def radius_error_cases(L):
    wb = L.b2d_radius_neighbors_workspace_bytes
    D = mwc.D
    m, n, k, nnz = 300, 500, 96, 12345
    cases = []
    for metric in (0, 1, 2, 10):
        cases.append(("count metric %d" % metric, "b2d_radius_neighbors_count",
                      [None, D, metric, D, k, D, k + 4, m, n, k, 2.5], wb(m, n, k, 0), True))
        cases.append(("fill metric %d" % metric, "b2d_radius_neighbors_fill",
                      [None, D, nnz, D, D, metric, D, k + 1, D, k, m, n, k, 2.5], wb(m, n, k, nnz), True))
    return cases


def main():
    L = mwc._lib.lib()
    out = mwc.record(L, radius_byte_queries, radius_error_cases)
    path = os.path.join(HERE, "radius_neighbors_workspace_contract.json")
    with open(path, "w") as f:   # one case per line, as the other fixtures
        f.write('{"bytes": {\n')
        f.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                           for fn, rows in out["bytes"].items()))
        f.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
