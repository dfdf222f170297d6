"""Generates tests/golden/hdbscan_rbc_workspace_contract.json (run without a GPU; the output is committed), in the format
and with the recorder of make_workspace_contract.py:
  bytes   b2d_hdbscan_rbc_workspace_bytes over m from 0 to 2^30 (around the 2^28-item sort portion), d from 1 to 4 and
          n_landmarks from 0 (ceil(sqrt(m))) to m + 1; plus negative arguments;
  errors  the fit for both metrics, both d and both selection methods given a null, short or misaligned workspace.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_workspace_contract as mwc  # noqa: E402
from make_single_linkage_rbc_workspace_contract import SL_DS, SL_MS  # noqa: E402


def hdb_byte_queries():
    q = [(m, d, nl) for m in SL_MS for d in SL_DS for nl in sorted({0, 1, 7, m, m + 1})] + \
        [(-1, 2, 0), (5, -2, 0), (5, 2, -1)]
    return {"b2d_hdbscan_rbc_workspace_bytes": q}


def hdb_error_cases(L):
    D = mwc.D
    m = 5000
    cases = []
    for metric in (4, 5):
        for d in (2, 3):
            for method in (0, 1):
                cases.append(("hdbscan metric %d d %d method %d" % (metric, d, method), "b2d_hdbscan_rbc_fit",
                              [None, metric, D, d + 1, m, d, 5, 10, 0.5, method, 0, 0, 7, D, D, D, D, D, D],
                              L.b2d_hdbscan_rbc_workspace_bytes(m, d, 0), True))
    return cases


def main():
    L = mwc._lib.lib()
    out = mwc.record(L, hdb_byte_queries, hdb_error_cases)
    path = os.path.join(HERE, "hdbscan_rbc_workspace_contract.json")
    with open(path, "w") as f:   # one case per line, as the other fixtures
        f.write('{"bytes": {\n')
        f.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                           for fn, rows in out["bytes"].items()))
        f.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
