"""DBSCAN on a given boolean adjacency A (numpy), by the rules b2d_dbscan_fit states (include/raft_b200.h):
deg(j) = #{i : A[i, j]} (the columns; A need not be symmetric), j is core iff deg(j) >= min_samples, core rows i and j
are linked iff A[i, j] or A[j, i], clusters are the components of the core rows numbered by their smallest row, and a
non-core row b takes the smallest cluster number of the core rows c with A[b, c], else -1.

Returns (labels int32 [m], core_sample_indices int32 [m] padded with -1, n_clusters)."""
import numpy as np


def dbscan_ref(A, min_samples):
    A = np.asarray(A, dtype=bool)
    m = A.shape[0]
    core = A.sum(axis=0) >= min_samples
    cidx = np.flatnonzero(core)
    # union-find over the core rows, hooking the larger root under the smaller
    parent = np.arange(m)

    def find(v):
        while parent[v] != v:
            parent[v] = parent[parent[v]]
            v = parent[v]
        return v

    sub = A[np.ix_(cidx, cidx)]
    ii, jj = np.nonzero(sub | sub.T)
    for a, b in zip(cidx[ii], cidx[jj]):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    roots = np.array([find(v) for v in cidx], dtype=np.int64)
    labels = np.full(m, -1, np.int64)
    num = {}
    for v, r in zip(cidx, roots):   # ascending rows: a cluster's number is fixed at its smallest row
        labels[v] = num.setdefault(r, len(num))
    for b in np.flatnonzero(~core):
        reach = labels[cidx[A[b, cidx]]]
        if reach.size:
            labels[b] = reach.min()
    csi = np.full(m, -1, np.int32)
    csi[:cidx.size] = cidx
    return labels.astype(np.int32), csi, len(num)


def dbscan_ref_edges(rows, cols, m, min_samples):
    """The same rules for an A given by its set entries (rows[e], cols[e]) -- for sizes where A does not fit as a dense
    matrix.  Components by scipy.sparse.csgraph over the core-core entries, taken as undirected."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    core = np.bincount(cols, minlength=m) >= min_samples
    both = core[rows] & core[cols]
    g = coo_matrix((np.ones(int(both.sum()), np.int8), (rows[both], cols[both])), shape=(m, m))
    _, comp = connected_components(g, directed=True, connection="weak")
    cidx = np.flatnonzero(core)
    # number the components of the core rows by their smallest core row
    first = np.full(m, m, np.int64)
    np.minimum.at(first, comp[cidx], cidx)
    roots = first[comp[cidx]]
    uniq = np.unique(roots)
    labels = np.full(m, -1, np.int64)
    labels[cidx] = np.searchsorted(uniq, roots)
    # border: the smallest label among the core columns of a non-core row
    hit = ~core[rows] & core[cols]
    best = np.full(m, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(best, rows[hit], labels[cols[hit]])
    nb = ~core & (best != np.iinfo(np.int64).max)
    labels[nb] = best[nb]
    csi = np.full(m, -1, np.int32)
    csi[:cidx.size] = cidx
    return labels.astype(np.int32), csi, int(uniq.size)
