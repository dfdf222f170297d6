"""Generates tests/golden/hdbscan_predict_model_contract.json (run without a GPU; the output is committed), in the format
of make_workspace_contract.py:
  bytes   b2d_hdbscan_rbc_model_bytes over m from 0 to 2^30 (around the 2^28-item sort portion), d from 1 to 4 and
          n_landmarks from 0 (ceil(sqrt(m))) to m + 1; plus negative arguments;
  errors  b2d_hdbscan_rbc_fit_model for both metrics, both d and both selection methods given a null, short or
          misaligned workspace (with a model), or a null or misaligned model (with a workspace).
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_workspace_contract as mwc  # noqa: E402
from make_single_linkage_rbc_workspace_contract import SL_DS, SL_MS  # noqa: E402


def model_byte_queries():
    q = [(m, d, nl) for m in SL_MS for d in SL_DS for nl in sorted({0, 1, 7, m, m + 1})] + \
        [(-1, 2, 0), (5, -2, 0), (5, 2, -1)]
    return {"b2d_hdbscan_rbc_model_bytes": q}


def model_error_cases(L):
    D, WS, ODD = mwc.D, mwc.WS, mwc.ODD
    m, out = 5000, []
    for metric in (4, 5):
        for d in (2, 3):
            for method in (0, 1):
                name = "hdbscan model metric %d d %d method %d" % (metric, d, method)
                args = [None, metric, D, d + 1, m, d, 5, 10, 0.5, method, 0, 0, 7, D, D, D, D, D, D]
                need = L.b2d_hdbscan_rbc_workspace_bytes(m, d, 0)
                for case, ws, nbytes, model in (("null", None, need, WS), ("short", WS, need - 1, WS),
                                                ("odd", ODD, need, WS), ("null model", WS, need, None),
                                                ("odd model", WS, need, ODD)):
                    a = args + [ws, nbytes, model]
                    rc = L.b2d_hdbscan_rbc_fit_model(*a)
                    if rc in (0, 2):
                        raise SystemExit("%s / %s: status %d -- the call got past validation" % (name, case, rc))
                    out.append({"name": name, "case": case, "fn": "b2d_hdbscan_rbc_fit_model", "args": a, "rc": rc,
                                "msg": L.b2d_last_error().decode()})
    return out


def main():
    L = mwc._lib.lib()
    out = mwc.record(L, model_byte_queries, lambda L: [])
    out["errors"] = model_error_cases(L)
    path = os.path.join(HERE, "hdbscan_predict_model_contract.json")
    with open(path, "w") as f:   # one case per line, as the other fixtures
        f.write('{"bytes": {\n')
        f.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                           for fn, rows in out["bytes"].items()))
        f.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
    print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
