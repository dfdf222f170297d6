"""Host references of radius_neighbors: the CSR of every pair within a radius, each row in the packed (distance, index) key
order of oracle.pack_minloc.

ref_csr64      fp64 distances (the semantics, pinned to sklearn in tests/test_radius_neighbors.py)
composition    the float32 matrix pairwise_distance returns, compared and ordered on the host: what the GPU tier compares the
               fused call with, bit for bit
"""
import numpy as np

import oracle

METRIC_IDS = {"sqeuclidean": 0, "euclidean": 1, "cosine": 2, "correlation": 10}


def dist64(q, x, metric):
    """fp64 distance matrix [m, n] of the queries q to the dataset rows x"""
    q, x = np.asarray(q, np.float64), np.asarray(x, np.float64)
    if metric == "correlation":
        q = q - q.mean(1, keepdims=True)
        x = x - x.mean(1, keepdims=True)
    if metric in ("cosine", "correlation"):
        with np.errstate(divide="ignore", invalid="ignore"):
            qn = q / np.linalg.norm(q, axis=1, keepdims=True)
            xn = x / np.linalg.norm(x, axis=1, keepdims=True)
        return 1.0 - qn @ xn.T
    d = (q * q).sum(1)[:, None] + (x * x).sum(1)[None, :] - 2.0 * (q @ x.T)
    d = np.maximum(d, 0.0)
    return np.sqrt(d) if metric == "euclidean" else d


def csr_from_dense(d, radius):
    """CSR (indptr, indices, distances) of the pairs d <= radius of a dense [m, n] matrix, rows in key order.  The key
    order is that of the float32 value: fp64 matrices are ordered by their float32 rounding, then by the fp64 value."""
    d = np.asarray(d)
    m, n = d.shape
    if not (radius >= 0):
        return np.zeros(m + 1, np.int64), np.zeros(0, np.int64), np.zeros(0, d.dtype)
    hit = d <= radius
    indptr = np.zeros(m + 1, np.int64)
    indptr[1:] = np.cumsum(hit.sum(1))
    indices, dists = [], []
    for i in range(m):
        j = np.nonzero(hit[i])[0]
        v = d[i, j]
        if d.dtype == np.float32:
            order = np.argsort(oracle.pack_minloc(v, j), kind="stable")
        else:
            order = np.lexsort((j, v))
        indices.append(j[order])
        dists.append(v[order])
    cat = (lambda a, t: np.concatenate(a).astype(t) if a else np.zeros(0, t))
    return indptr, cat(indices, np.int64), cat(dists, d.dtype)


def ref_csr64(q, x, radius, metric):
    """the fp64 CSR of the queries q against x (no self-pair rule: a zero distance is what fp64 gives)"""
    return csr_from_dense(dist64(q, x, metric), radius)


def composition(d32, radius):
    """the CSR the fused call must equal bit for bit: the float32 matrix of pairwise_distance, d <= radius, each row sorted
    by oracle.pack_minloc(d, j)"""
    d32 = np.asarray(d32, np.float32)
    return csr_from_dense(d32, np.float32(radius) if radius == radius else radius)
