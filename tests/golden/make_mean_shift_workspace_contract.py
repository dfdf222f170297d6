"""Generates tests/golden/mean_shift_workspace_contract.json (run without a GPU; the output is committed), in the format
and with the recorder of make_workspace_contract.py:
  bytes   b2d_mean_shift_fit_workspace_bytes over data sizes around the 2048-row chunk and the 16-byte adjacency pitch,
          every k of the other fixtures, no caller seeds or fewer / more seeds than rows, and batch bounds from the
          default (0) through one 128-seed batch to more than the whole adjacency, plus negative arguments;
  errors  the call with rows, bin or caller seeds (pitched) given a null, short or misaligned workspace.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_workspace_contract as mwc  # noqa: E402

MS_NS = [1, 15, 16, 17, 2047, 2048, 2049, 100000]
MS_SEEDS = [0, 1, 129, 300000]
MS_BATCH = [0, 1, 1 << 20, 1 << 40]


def ms_byte_queries():
    q = [(n, k, s, b) for n in MS_NS for k in mwc.KS for s in MS_SEEDS for b in MS_BATCH] + \
        [(-1, 5, 0, 0), (5, -1, 0, 0), (5, 5, -1, 0), (5, 5, 0, -1)]
    return {"b2d_mean_shift_fit_workspace_bytes": q}


def ms_error_cases(L):
    wb = L.b2d_mean_shift_fit_workspace_bytes
    D = mwc.D
    n, k = 500, 96
    return [
        ("rows as seeds", "b2d_mean_shift_fit", [None, D, k, n, k, 1.5, None, k, 0, 0, 1, 1, 300, 0, D, D, D, D],
         wb(n, k, 0, 0), True),
        ("bin seeding", "b2d_mean_shift_fit", [None, D, k, n, k, 1.5, None, k, 0, 1, 3, 0, 10, 1 << 20, D, D, D, D],
         wb(n, k, 0, 1 << 20), True),
        ("pitched seeds", "b2d_mean_shift_fit", [None, D, k + 4, n, k, 1.5, D, k + 8, 40, 0, 1, 1, 0, 0, D, D, D, None],
         wb(n, k, 40, 0), True),
        ("more seeds than rows", "b2d_mean_shift_fit", [None, D, k, n, k, 0.5, D, k, 2 * n, 1, 1, 1, 1, 0, D, D, D, D],
         wb(n, k, 2 * n, 0), True),
    ]


def main():
    L = mwc._lib.lib()
    out = mwc.record(L, ms_byte_queries, ms_error_cases)
    path = os.path.join(HERE, "mean_shift_workspace_contract.json")
    with open(path, "w") as f:   # one case per line, as the other fixtures
        f.write('{"bytes": {\n')
        f.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                           for fn, rows in out["bytes"].items()))
        f.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
