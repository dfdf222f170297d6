"""Generates the workspace-contract fixtures under tests/golden (run here, without a GPU; the outputs are committed).

Each fixture pins the workspace contract of a group of C ABI entry points:
  bytes   every *_workspace_bytes query of the group over a grid that reaches every branch of its workspace layouts;
  errors  (status, b2d_last_error()) of every entry point of the group that takes a workspace, given a null workspace,
          one byte too few at an aligned address, or the full size at an odd address -- with every other argument valid.
The fixtures:
  workspace_contract.json                 distances, nearest neighbours, select_k and the stats;
  kmeans_workspace_contract.json          k-means, over row counts past the histogram cap and 1 to 10^5 clusters;
  gram_workspace_contract.json            gram_matrix for every kernel id (and two invalid ones) and dtype;
  single_linkage_workspace_contract.json  single_linkage over row counts from 1 to 10^6 (around the 2048-row sort blocks
                                          and the 2^20-row tile-class cap) and c from -5 to 60 (n_nb from 2 to past 64),
                                          and the edge-list MST;
  dbscan_workspace_contract.json          dbscan over row counts around the 16-column adjacency pitch and the 256-column
                                          batch step, every k, and batch sizes from the 2^30 default (0) through the
                                          256-column floor (1) to one batch of every column; null, short or misaligned
                                          workspaces for the euclidean, cosine (batched, optional outputs null) and
                                          sqeuclidean (NaN eps) fits.
Pointers are fake addresses: the calls must fail in validation, before anything reaches the device.  A case that
returns B2D_OK or B2D_ERR_CUDA got past validation, so it is refused rather than recorded.  The library is the one
raft_b200._lib loads (RAFT_B200_LIB selects another build of the same ABI).
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from raft_b200 import _lib  # noqa: E402

METRICS = list(range(-1, 21))                   # every DistanceType value, 13 (Haversine) and two out of range
DTYPES = [0, 1, 2, 3]                           # F32, F16, F64 and one unknown
KS = [1, 31, 32, 33, 128, 129, 320, 321]
NEG = [(-1, 29, 32), (37, -1, 32), (37, 29, -1)]
NN_N = [1000, (1 << 20) - 1, 1 << 20, (1 << 20) + 1]   # around the 2^20-row chunk of the screened search
BIG_M = 1 << 24                                 # 128 m + 2^19 > 2^31 - 1: the candidate list is clamped


def byte_queries():
    q = {}
    edges = [(0, 29, 32), (37, 0, 32), (37, 29, 0)] + NEG
    shapes = [(37, 29, k) for k in KS] + edges + [(BIG_M, 1000, 96)]
    # every metric and dtype at one shape and the edges; every k for an expanded and an unexpanded metric
    q["b2d_pairwise_workspace_bytes"] = [(mt, dt) + s for mt in METRICS for dt in DTYPES for s in [(37, 29, 33)] + edges] + \
                                        [(mt, dt) + s for mt in (0, 3) for dt in DTYPES for s in shapes]
    nn = [(m, n, k) for m in (1, 100) for n in NN_N for k in KS] + \
         [(0, 29, 32), (37, 0, 32), (37, 29, 0), (BIG_M, 1000, 96), (BIG_M, 1 << 20, 128)] + NEG
    q["b2d_fused_l2_nn_workspace_bytes"] = nn
    q["b2d_eps_neighbors_l2sq_workspace_bytes"] = [s for s in shapes] + [(1000, 1 << 20, 128)]
    # G = 0, G <= m / 32 and G > m / 32
    q["b2d_masked_l2_nn_workspace_bytes"] = [(m, n, k, g) for m, n in ((1, 1), (1000, 3000), (4096, 777))
                                             for k in (1, 32, 129, 320) for g in (0, 1, 20, 200)] + \
                                            [(-1, 5, 8, 1), (5, -1, 8, 1), (5, 5, -1, 1), (5, 5, 8, -1), (0, 5, 8, 3)]
    q["b2d_knn_l2_workspace_bytes"] = [(m, n, k, kk) for m in (1, 1000, BIG_M) for n in (64, 5000)
                                       for k in (1, 32, 129, 320) for kk in (1, 64)] + \
                                      [(100, 100, 32, 0), (100, 100, 32, 65), (-1, 5, 8, 1), (5, -1, 8, 1), (5, 5, -1, 1),
                                       (0, 5, 8, 3)]
    # default (0) and explicit chunk rows; L2Expanded, L1 (no pairwise scratch), Haversine (not supported)
    q["b2d_silhouette_score_workspace_bytes"] = [(n, k, nl, mt, c) for n in (0, 1000, 300000) for k in (3, 129)
                                                 for nl in (1, 50) for mt in (0, 3, 13)
                                                 for c in (0, 1, 1000, 1 << 20)] + \
                                                [(-1, 3, 2, 0, 0), (10, -1, 2, 0, 0), (10, 3, 0, 0, 0), (10, 3, 2, 0, -1)]
    q["b2d_trustworthiness_score_workspace_bytes"] = [(n, m, d, kk, mt, b) for n in (0, 100, 300000) for m in (8, 129)
                                                      for d in (2, 64) for kk in (1, 63) for mt in (0, 2, 13, 3)
                                                      for b in (0, 1000)] + \
                                                     [(100, 8, 2, 0, 0, 0), (100, 8, 2, 64, 0, 0), (-1, 8, 2, 5, 0, 0),
                                                      (100, -1, 2, 5, 0, 0), (100, 8, -1, 5, 0, 0), (100, 8, 2, 5, 0, -1)]
    # sort-row, radix-row (list in shared memory, list + cub), split (shared-memory sort, cub), cub in several batches
    q["b2d_select_k_workspace_bytes"] = [
        (100000, 1024, 32), (4, 2048, 2048), (16384, 100000, 1024), (264, 40000, 10), (300, 100000, 5000),
        (1, 1 << 28, 1024), (2, 200000, 5), (263, 40000, 10), (1, 1 << 20, 5000), (2000, 1 << 20, 1 << 20),
        (0, 5, 3), (0, 5, 0), (1, 5, 0), (1, 5, 6), (-1, 5, 1), (1, 1 << 31, 1), (1 << 31, 10, 1)]
    return q


D = 0x10000000                # fake data pointer
WS = 0x20000000               # fake workspace, 256-byte aligned
ODD = WS + 1                  # fake workspace at an odd address


def error_cases(L):
    """(name, function, arguments before the workspace pair, bytes needed, has an alignment check)"""
    pw = L.b2d_pairwise_workspace_bytes
    nn = L.b2d_fused_l2_nn_workspace_bytes
    m, n, k = 300, 500, 96
    return [
        ("pairwise L2Expanded f32", "b2d_pairwise_distance", [None, 0, 0, D, k, D, k, D, n, m, n, k, 1, 2.0], pw(0, 0, m, n, k), True),
        ("pairwise Cosine f16 col-major", "b2d_pairwise_distance", [None, 2, 1, D, m, D, n, D, m, m, n, k, 0, 2.0],
         pw(2, 1, n, m, k), True),
        ("pairwise L1 f64", "b2d_pairwise_distance", [None, 3, 2, D, k, D, k, D, n, m, n, k, 1, 2.0], pw(3, 2, m, n, k), False),
        ("fused_l2_nn", "b2d_fused_l2_nn", [None, D, D, k, D, k, None, None, m, n, k, 1, 1], nn(m, n, k), True),
        ("fused_distance_nn L2SqrtExpanded", "b2d_fused_distance_nn", [None, D, 1, D, k, D, k, None, None, m, n, k, 1],
         nn(m, n, k), True),
        ("fused_distance_nn CosineExpanded", "b2d_fused_distance_nn", [None, D, 2, D, k, D, k, None, None, m, n, k, 1],
         nn(m, n, k), True),
        ("fused_distance_nn CorrelationExpanded", "b2d_fused_distance_nn", [None, D, 10, D, k, D, k, None, None, m, n, k, 0],
         nn(m, n, k), True),
        ("fused_l2_nn_keys", "b2d_fused_l2_nn_keys", [None, D, D, k, D, k, None, None, m, n, k, 7, 1], nn(m, n, k), True),
        ("fused_l2_nn_finalize", "b2d_fused_l2_nn_finalize", [None, D, D, m, 0], 1024 + 4 * m, False),
        ("masked_l2_nn", "b2d_masked_l2_nn", [None, D, D, k, D, k, None, None, D, 16, D, 9, m, n, k, 0, 1],
         L.b2d_masked_l2_nn_workspace_bytes(m, n, k, 9), True),
        ("masked_l2_nn G=0", "b2d_masked_l2_nn", [None, D, D, k, D, k, None, None, None, 0, None, 0, m, n, k, 0, 1],
         L.b2d_masked_l2_nn_workspace_bytes(m, n, k, 0), True),
        ("knn CosineExpanded", "b2d_knn", [None, D, D, 2, D, k, D, k, m, n, k, 10], L.b2d_knn_l2_workspace_bytes(m, n, k, 10),
         True),
        ("knn_l2 sqrt", "b2d_knn_l2", [None, D, D, D, k, D, k, m, n, k, 64, 1], L.b2d_knn_l2_workspace_bytes(m, n, k, 64),
         True),
        ("silhouette L2Expanded", "b2d_silhouette_score", [None, D, D, D, k, D, n, k, 7, 0, 2.0, 0],
         L.b2d_silhouette_score_workspace_bytes(n, k, 7, 0, 0), True),
        ("silhouette L1 chunked", "b2d_silhouette_score", [None, D, None, D, k, D, n, k, 7, 3, 2.0, 128],
         L.b2d_silhouette_score_workspace_bytes(n, k, 7, 3, 128), True),
        ("trustworthiness L2SqrtUnexpanded", "b2d_trustworthiness_score", [None, D, D, k, D, 2, n, k, 2, 5, 5, 0],
         L.b2d_trustworthiness_score_workspace_bytes(n, k, 2, 5, 5, 0), True),
        ("select_k split", "b2d_select_k", [None, D, 200000, None, 2, 200000, 5, 1, D, D],
         L.b2d_select_k_workspace_bytes(2, 200000, 5), True),
        ("select_k radix-row cub", "b2d_select_k", [None, D, 100000, D, 300, 100000, 5000, 0, D, D],
         L.b2d_select_k_workspace_bytes(300, 100000, 5000), True),
        ("eps", "b2d_eps_neighbors_l2sq", [None, D, n, D, 0, 1, D, k, D, k, m, n, k, 4.0], L.b2d_eps_neighbors_l2sq_workspace_bytes(m, n, k),
         True),
    ]


KM_MS = [1, 37, 2048, 2049, 100000, 1000000]
KM_NCS = [1, 17, 1000, 100000]
KM_NEG = [(-1, 32, 4), (37, -1, 4), (37, 32, -1)]


def kmeans_byte_queries():
    shapes = [(m, k, nc) for m in KM_MS for k in KS for nc in KM_NCS] + [(0, 32, 0), (37, 0, 4)] + KM_NEG
    return {"b2d_kmeans_workspace_bytes": shapes}


def kmeans_error_cases(L):
    wb = L.b2d_kmeans_workspace_bytes
    m, k, nc = 5000, 96, 40
    return [
        ("fit array", "b2d_kmeans_fit", [None, nc, 20, 1e-4, 2, 1, 0, 0, D, k, None, m, k, D, D, D], wb(m, k, nc), True),
        ("fit k-means++ weighted n_init=3", "b2d_kmeans_fit", [None, nc, 20, 1e-4, 0, 3, 7, 1, D, k, D, m, k, D, D, D],
         wb(m, k, nc), True),
        ("predict", "b2d_kmeans_predict", [None, D, k, None, m, k, D, nc, D, D, 1], wb(m, k, nc), True),
        ("update_centroids", "b2d_kmeans_update_centroids", [None, D, k, D, D, m, k, D, nc, D, None], wb(m, k, nc), True),
        ("init_plus_plus", "b2d_kmeans_init_plus_plus", [None, D, k, None, m, k, nc, 3, D], wb(m, k, nc), True),
    ]


GRAM_KERNEL_IDS = list(range(-1, 5))   # LINEAR, POLYNOMIAL, RBF, TANH and one invalid id on either side


def gram_byte_queries():
    edges = [(0, 29, 32), (37, 0, 32), (37, 29, 0)] + NEG
    shapes = [(37, 29, k) for k in KS] + edges + [(BIG_M, 1000, 96), (1000, 1 << 20, 128)]
    return {"b2d_gram_matrix_workspace_bytes": [(kr, dt) + s for kr in GRAM_KERNEL_IDS for dt in DTYPES for s in shapes]}


def gram_error_cases(L):
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


SL_MS = [1, 2, 37, 2048, 2049, 100000, (1 << 20) + 1, 1000000]
SL_CS = [-5, 1, 15, 45, 60]
MST_NS = [0, 1, 1000, 1000000]
MST_ES = [0, 5000, 10 ** 7]


def single_linkage_byte_queries():
    sl = [(m, d, c) for m in SL_MS for d in KS for c in SL_CS] + [(0, 32, 15), (-1, 32, 15), (37, -1, 15)]
    mst = [(n, e) for n in MST_NS for e in MST_ES] + [(-1, 10), (10, -1)]
    return {"b2d_single_linkage_workspace_bytes": sl, "b2d_mst_workspace_bytes": mst}


def single_linkage_error_cases(L):
    m, d, n, e = 5000, 96, 3000, 20000
    return [
        ("single_linkage euclidean", "b2d_single_linkage", [None, 1, D, d, m, d, 15, 7, D, D, D, D, D],
         L.b2d_single_linkage_workspace_bytes(m, d, 15), True),
        ("single_linkage sqeuclidean c=40", "b2d_single_linkage", [None, 0, D, d + 3, m, d, 40, 1, D, D, D, D, D],
         L.b2d_single_linkage_workspace_bytes(m, d, 40), True),
        ("mst", "b2d_mst", [None, D, D, D, n, e, D, D, D, D, D], L.b2d_mst_workspace_bytes(n, e), True),
    ]


DB_MS = [1, 15, 16, 256, 257, 32768, 100000, 1000000]
DB_BATCH = [0, 1, 1 << 20, 1 << 26, (1 << 30) + 1, 1 << 40]


def dbscan_byte_queries():
    q = [(m, d, b) for m in DB_MS for d in KS for b in DB_BATCH] + \
        [(0, 32, 0), (-1, 32, 0), (37, -1, 0), (37, 32, -1)]
    return {"b2d_dbscan_workspace_bytes": q}


def dbscan_error_cases(L):
    m, d = 5000, 96
    return [
        ("dbscan euclidean", "b2d_dbscan_fit", [None, 1, D, d, m, d, 0.5, 5, 0, D, D, D],
         L.b2d_dbscan_workspace_bytes(m, d, 0), True),
        ("dbscan cosine batched", "b2d_dbscan_fit", [None, 2, D, d + 3, m, d, 0.1, 1, 1 << 20, D, None, None],
         L.b2d_dbscan_workspace_bytes(m, d, 1 << 20), True),
        ("dbscan sqeuclidean NaN eps", "b2d_dbscan_fit", [None, 0, D, d, m, d, float("nan"), 50, 12345, D, D, None],
         L.b2d_dbscan_workspace_bytes(m, d, 12345), True),
    ]


FIXTURES = {   # file -> (size queries, error cases)
    "workspace_contract.json": (byte_queries, error_cases),
    "kmeans_workspace_contract.json": (kmeans_byte_queries, kmeans_error_cases),
    "gram_workspace_contract.json": (gram_byte_queries, gram_error_cases),
    "single_linkage_workspace_contract.json": (single_linkage_byte_queries, single_linkage_error_cases),
    "dbscan_workspace_contract.json": (dbscan_byte_queries, dbscan_error_cases),
}


def record(L, queries, cases):
    out = {"bytes": {}, "errors": []}
    for fn, args in queries().items():
        out["bytes"][fn] = [list(a) + [getattr(L, fn)(*a)] for a in args]
    for name, fn, args, need, aligned in cases(L):
        assert 0 < need < 2 ** 63, (name, need)
        variants = [("null", None, need), ("short", WS, need - 1)] + ([("odd", ODD, need)] if aligned else [])
        for case, ws, nbytes in variants:
            a = args + [ws, nbytes]
            rc = getattr(L, fn)(*a)
            if rc in (_lib.B2D_OK, _lib.B2D_ERR_CUDA):
                raise SystemExit(f"{name} / {case}: status {rc} -- the call got past validation; not recorded")
            out["errors"].append({"name": name, "case": case, "fn": fn, "args": a, "rc": rc,
                                  "msg": L.b2d_last_error().decode()})
    return out


def main():
    L = _lib.lib()
    for name, (queries, cases) in FIXTURES.items():
        out = record(L, queries, cases)
        path = os.path.join(HERE, name)
        with open(path, "w") as f:   # one case per line, so that a change to the contract reads as a short diff
            f.write('{"bytes": {\n')
            f.write(",\n".join(json.dumps(fn) + ": [\n" + ",\n".join(json.dumps(r) for r in rows) + "]"
                               for fn, rows in out["bytes"].items()))
            f.write('},\n"errors": [\n' + ",\n".join(json.dumps(e) for e in out["errors"]) + "]}\n")
        print("wrote", path, sum(map(len, out["bytes"].values())), "size queries,", len(out["errors"]), "error cases")


if __name__ == "__main__":
    main()
