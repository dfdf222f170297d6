"""fp64 restatement of raft_b200's single_linkage (include/raft_b200.h, b2d_single_linkage; DESIGN.md K13) and of its
minimum spanning forest (b2d_mst), for the tests.

Edge order: edge e of weight w has the key (w, e).  For float32 weights w is compared by the ordered bits of the
float (nn_key.cuh ordered_bits: -0.0 before +0.0, the order of the device), for float64 by value.  Kruskal under this
strict order gives the unique forest the device's Borůvka builds."""
import numpy as np


def ordered_bits(w):
    b = np.ascontiguousarray(w, np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, b ^ 0x7FFFFFFF, b)


def edge_order(w):
    w = np.asarray(w)
    key = ordered_bits(w) if w.dtype == np.float32 else w
    return np.lexsort((np.arange(len(w)), key))


def _find(p, v):
    while p[v] != v:
        p[v] = p[p[v]]
        v = p[v]
    return v


def kruskal(src, dst, w, n):
    """Minimum spanning forest of the edge list on n vertices: (positions of the forest edges in key order, colour),
    colour[v] = the smallest vertex of v's tree.  Edges with an endpoint outside [0, n) are ignored."""
    p = list(range(n))
    chosen = []
    for e in edge_order(w):
        a, b = int(src[e]), int(dst[e])
        if not (0 <= a < n and 0 <= b < n):
            continue
        ra, rb = _find(p, a), _find(p, b)
        if ra != rb:
            p[max(ra, rb)] = min(ra, rb)
            chosen.append(int(e))
    colour = np.array([_find(p, v) for v in range(n)], np.int64)   # the root is the smallest vertex of its tree
    return np.array(chosen, np.int64), colour


def n_neighbors(m, c=15):
    return min(m, max(2, int(np.floor(np.log2(m))) + c)) if m >= 1 else 0


def knn_exact(x, k):
    """fp64 brute-force kNN of x against itself: (idx [m, k], squared distances [m, k]) in (distance, index) order."""
    x = np.asarray(x, np.float64)
    d2 = ((x[:, None, :] - x[None, :, :]) ** 2).sum(-1)
    idx = np.stack([np.lexsort((np.arange(len(x)), row))[:k] for row in d2])
    return idx, np.take_along_axis(d2, idx, 1)


def knn_edges(idx, dist):
    """Step 1: edge i n_nb + s = (i, idx[i, s], dist[i, s]); a row's edge to itself is a self-loop (never chosen)."""
    m, k = idx.shape
    src = np.repeat(np.arange(m), k)
    dst = np.where(idx.reshape(-1) < 0, src, idx.reshape(-1))
    return src, dst, np.asarray(dist).reshape(-1)


def connect_edges(x, colour):
    """Step 4 in fp64: for every tree, the edge from its row i of smallest (d_i, i) to that row's nearest row of another
    tree, d_i the squared distance; trees in order of their smallest row.  colour[v] is the smallest row of v's tree.
    Among equidistant nearest rows the first in (smallest row of its tree, row) order wins, not the smallest row: the
    device's arg-min runs over the rows sorted by tree and takes the smallest sorted position."""
    x = np.asarray(x, np.float64)
    colour = np.asarray(colour)
    order = np.lexsort((np.arange(len(x)), colour))   # the candidates in (smallest row of their tree, row) order
    xo, co = x[order], colour[order]
    nx = (x * x).sum(1)
    j = np.zeros(len(x), np.int64)
    di = np.zeros(len(x))
    for r0 in range(0, len(x), 1024):   # row blocks: m x m distances are never held at once
        d2 = np.maximum(nx[r0:r0 + 1024, None] + nx[order][None, :] - 2 * x[r0:r0 + 1024] @ xo.T, 0)
        d2[colour[r0:r0 + 1024, None] == co[None, :]] = np.inf
        j[r0:r0 + 1024] = order[d2.argmin(1)]
        di[r0:r0 + 1024] = d2.min(1)
    out = []
    for g in np.unique(colour):
        rows = np.flatnonzero(colour == g)
        i = rows[np.lexsort((rows, di[rows]))[0]]
        out.append((i, j[i], di[i]))
    return [np.array(v) for v in zip(*out)]


def dendrogram(src, dst, w, m, n_clusters, sqrt):
    """Step 5: merges of the forest edges (given in key order) -> children [m-1, 2], deltas, sizes, labels."""
    p, cid, size = list(range(m)), list(range(m)), [1] * m
    children = np.zeros((m - 1, 2), np.int64)
    sizes = np.zeros(m - 1, np.int64)
    labels = None
    for t in range(m - 1):
        if t == m - n_clusters:
            labels = np.array([_find(p, i) for i in range(m)])
        a, b = _find(p, int(src[t])), _find(p, int(dst[t]))
        assert a != b
        children[t] = sorted((cid[a], cid[b]))
        p[b] = a
        size[a] += size[b]
        sizes[t] = size[a]
        cid[a] = m + t
    if labels is None:
        labels = np.array([_find(p, i) for i in range(m)])
    _, first = np.unique(labels, return_index=True)
    rank = {labels[f]: r for r, f in enumerate(sorted(first))}
    deltas = np.sqrt(w) if sqrt else np.asarray(w)
    return children, deltas, sizes, np.array([rank[v] for v in labels], np.int64)


def single_linkage_from_knn(x, idx, dist, n_clusters, sqrt=True):
    """Steps 2-5 given the kNN output (idx, squared dist); connect_components in fp64 when the graph is disconnected.
    Returns (children, deltas, sizes, labels, n_connected_components)."""
    m = len(x)
    src, dst, w = knn_edges(idx, dist)
    chosen, colour = kruskal(src, dst, w, m)
    ncomp = len(np.unique(colour))
    while len(np.unique(colour)) > 1:
        cs, cd, cw = connect_edges(x, colour)
        src, dst = np.concatenate([src, cs]), np.concatenate([dst, cd])
        w = np.concatenate([w, cw.astype(w.dtype)])
        chosen, colour = kruskal(src, dst, w, m)
    ch, de, sz, lab = dendrogram(src[chosen], dst[chosen], w[chosen], m, n_clusters, sqrt)
    return ch, de, sz, lab, ncomp


def single_linkage(x, n_clusters, c=15, sqrt=True):
    """The whole algorithm in fp64 with an exact kNN."""
    idx, dist = knn_exact(x, n_neighbors(len(x), c))
    return single_linkage_from_knn(x, idx, dist, n_clusters, sqrt)


def canonical_labels(labels):
    """Any labelling renumbered in order of each cluster's smallest row (the numbering of single_linkage)."""
    labels = np.asarray(labels)
    _, first = np.unique(labels, return_index=True)
    rank = {labels[f]: r for r, f in enumerate(sorted(first))}
    return np.array([rank[v] for v in labels], np.int64)
