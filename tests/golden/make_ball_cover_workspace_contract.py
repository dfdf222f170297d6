"""Generates tests/golden/ball_cover_workspace_contract.json (run without a GPU; the output is committed), in the format
and with the recorder of make_workspace_contract.py:
  bytes   b2d_ball_cover_index_bytes and b2d_ball_cover_build_workspace_bytes over n from 1 to 2^31 - 1 (around the
          2^28-item sort portion), d from 1 to 4 and n_landmarks from 0 (ceil(sqrt(n))) to n + 1; and
          b2d_ball_cover_eps_workspace_bytes over row counts around the 64-row scan bound and nnz from 0 (the count
          call) to 2^31 - 1; plus negative arguments;
  errors  the build, eps count and eps fill calls of both metrics and both d given a null, short or misaligned workspace.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_workspace_contract as mwc  # noqa: E402

BC_NS = [1, 2, 63, 1000, 100003, 1 << 28, (1 << 28) + 1, (1 << 31) - 1, 1 << 31]
BC_DS = [1, 2, 3, 4]
BC_MS = [0, 1, 63, 64, 65, 100000, (1 << 31) - 1]
BC_NNZ = [0, 1, 1000, (1 << 31) - 1]


def bc_byte_queries():
    idx = [(n, d, nl) for n in BC_NS for d in BC_DS for nl in sorted({0, 1, 7, n, n + 1})] + \
          [(0, 2, 0), (-1, 2, 0), (5, -2, 0), (5, 2, -1)]
    eps = [(m, z) for m in BC_MS for z in BC_NNZ] + [(-1, 0), (5, -1)]
    return {"b2d_ball_cover_index_bytes": idx, "b2d_ball_cover_build_workspace_bytes": idx,
            "b2d_ball_cover_eps_workspace_bytes": eps}


def bc_error_cases(L):
    D = mwc.D
    n, m, nnz = 5000, 300, 12345
    cases = []
    for metric in (4, 5):
        for d in (2, 3):
            cases.append(("build metric %d d %d" % (metric, d), "b2d_ball_cover_build",
                          [None, D, D, d + 1, n, d, metric, 0, 7], L.b2d_ball_cover_build_workspace_bytes(n, d, 0), True))
            cases.append(("eps_count metric %d d %d" % (metric, d), "b2d_ball_cover_eps_count",
                          [None, D, D, n, d, metric, 0, D, d, m, 0.5], L.b2d_ball_cover_eps_workspace_bytes(m, 0), True))
            cases.append(("eps_fill metric %d d %d" % (metric, d), "b2d_ball_cover_eps_fill",
                          [None, D, nnz, D, D, D, n, d, metric, 0, D, d, m, 0.5],
                          L.b2d_ball_cover_eps_workspace_bytes(m, nnz), True))
    return cases


def main():
    L = mwc._lib.lib()
    out = mwc.record(L, bc_byte_queries, bc_error_cases)
    path = os.path.join(HERE, "ball_cover_workspace_contract.json")
    with open(path, "w") as f:   # one case per line, as the other fixtures
        f.write('{"bytes": {\n')
        f.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                           for fn, rows in out["bytes"].items()))
        f.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
