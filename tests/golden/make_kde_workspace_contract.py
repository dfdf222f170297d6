"""Generates tests/golden/kde_workspace_contract.json (run without a GPU; the output is committed), in the format and with
the recorder of make_workspace_contract.py:
  bytes   b2d_kde_workspace_bytes over row counts around the 1 GiB partials budget of the default slab, dataset sizes
          around the 256-column y block and the 8192-row weight blocks, every k of the other fixtures, and batch_cols
          from the default (0) through one y block to more than n, plus negative arguments;
  errors  the call for every kernel, with and without weights and with a pitched dataset, given a null, short or
          misaligned workspace.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_workspace_contract as mwc  # noqa: E402

KDE_MS = [0, 1, 127, 128, 129, 100000, 1 << 20, (1 << 31) - 1]
KDE_NS = [1, 255, 256, 257, 8193, 100000]
KDE_BATCH = [0, 1, 256, 257, 1 << 20]


def kde_byte_queries():
    q = [(m, n, k, b) for m in KDE_MS for n in KDE_NS for k in mwc.KS for b in KDE_BATCH] + \
        [(-1, 5, 8, 0), (5, -1, 8, 0), (5, 5, -1, 0), (5, 5, 8, -1)]
    return {"b2d_kde_workspace_bytes": q}


def kde_error_cases(L):
    wb = L.b2d_kde_workspace_bytes
    D = mwc.D
    m, n, k = 300, 500, 96
    cases = []
    for kernel in range(6):
        cases.append(("kernel %d" % kernel, "b2d_kde_score_samples",
                      [None, kernel, 0.5, D, k, None, D, k, m, n, k, 0, D], wb(m, n, k, 0), True))
    cases.append(("gaussian weighted pitched batch_cols=300", "b2d_kde_score_samples",
                  [None, 0, 2.0, D, k + 4, D, D, k, m, n, k, 300, D], wb(m, n, k, 300), True))
    return cases


def main():
    L = mwc._lib.lib()
    out = mwc.record(L, kde_byte_queries, kde_error_cases)
    path = os.path.join(HERE, "kde_workspace_contract.json")
    with open(path, "w") as f:   # one case per line, as the other fixtures
        f.write('{"bytes": {\n')
        f.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                           for fn, rows in out["bytes"].items()))
        f.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
