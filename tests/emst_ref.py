"""The oracle of the exact single linkage on the ball cover (include/raft_b200.h, b2d_emst_rbc / b2d_single_linkage_rbc;
DESIGN.md K21): Kruskal over every pair i < j, enumerated in row-major order, with the float32 pair value of
tests/ball_cover_ref.dist (term by term, each operation rounded on its own).  kruskal orders by (w, position), and the
position of (i, j) grows with i, then j, so its order is exactly the contract's (s, min row, max row).  The loop here is
single_linkage_ref.kruskal's, ending once the tree is complete (tests/test_single_linkage_rbc.py checks that the two
agree)."""
import numpy as np
import torch

import ball_cover_ref as bref
from single_linkage_ref import _find, dendrogram, edge_order


def pair_values(x):
    """(src, dst, s) of every pair i < j of the float32 rows x (numpy [m, d]), row-major"""
    xt = torch.from_numpy(np.ascontiguousarray(x, np.float32))
    s = bref.dist(xt, xt, "sqeuclidean").numpy()
    i, j = np.triu_indices(len(x), 1)
    return i, j, s[i, j]


def kruskal_tree(src, dst, w, n):
    """single_linkage_ref.kruskal's positions of the tree edges, for a connected graph, stopping at n - 1 edges"""
    p = list(range(n))
    chosen = []
    for e in edge_order(w):
        if len(chosen) == n - 1:
            break
        ra, rb = _find(p, int(src[e])), _find(p, int(dst[e]))
        if ra != rb:
            p[max(ra, rb)] = min(ra, rb)
            chosen.append(int(e))
    return np.array(chosen, np.int64)


def emst(x, metric="sqeuclidean"):
    """(src, dst, w) of the tree in the contract's order: src < dst, w = s, or its correctly rounded root for
    "euclidean" (float32 sqrt is correctly rounded)"""
    src, dst, s = pair_values(x)
    chosen = kruskal_tree(src, dst, s, len(x))
    w = s[chosen]
    if metric == "euclidean":
        w = np.sqrt(w, dtype=np.float32)
    return src[chosen].astype(np.int32), dst[chosen].astype(np.int32), w.astype(np.float32)


def linkage(tree, n_clusters, metric="sqeuclidean"):
    """(children, deltas, sizes, labels) of the merges of a tree emst returned (single_linkage_ref.dendrogram):
    deltas are its weights"""
    src, dst, w = tree
    ch, de, sz, lab = dendrogram(src, dst, w, len(src) + 1, n_clusters, False)
    return ch.astype(np.int32), np.asarray(de, np.float32), sz.astype(np.int32), lab.astype(np.int32)


def single_linkage(x, n_clusters, metric="sqeuclidean"):
    return linkage(emst(x, metric), n_clusters, metric)
