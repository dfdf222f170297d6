"""raft::cluster::kmeans_balanced -- hierarchical balanced k-means on the fused L2 arg-min ([RECALLED]
raft::cluster::kmeans_balanced: fit, predict, fit_predict).  Dispatches through the C ABI (include/raft_b200.h:
b2d_kmeans_balanced_fit; prediction is b2d_kmeans_predict).  sqrt(n_clusters) mesoclusters, the fine clusters allocated
to them by size and fitted all at once on the masked arg-min, then a short pass over all centroids.  Results are
bit-identical from run to run.  Not re-exported at package level, where ``fit`` and ``predict`` mean k-means."""
from __future__ import annotations

import torch

from .. import _lib
from ..common import auto_convert_output, auto_sync_handle, cai_wrapper, device_ndarray
from .kmeans import _centroids_out, _matrix, _new, _ws


class KMeansBalancedParams:
    """``n_iters``: balanced-EM iterations of the mesocluster and fine stages (the final pass runs
    max(n_iters // 10, 2)).  ``seed`` keys the draws of the balancing step.  Only ``metric="sqeuclidean"``
    (L2Expanded) is supported; anything else raises LogicError."""

    def __init__(self, n_iters=20, metric="sqeuclidean", seed=0):
        if metric not in ("sqeuclidean", "L2Expanded"):
            raise _lib.LogicError("kmeans_balanced supports the sqeuclidean (L2Expanded) metric only, got %r" % (metric,))
        self.n_iters = int(n_iters)
        if self.n_iters < 1:
            raise ValueError("n_iters must be >= 1, got %r" % (n_iters,))
        self.metric = metric
        self.seed = int(seed)


def _fit(params, X, n_clusters, centroids, want_labels, handle):
    x = _matrix(X, "X")
    m, k = x.shape
    if n_clusters is None:
        if centroids is None:
            raise ValueError("n_clusters or centroids must be given")
        n_clusters = cai_wrapper(centroids).shape[0]
    nc = int(n_clusters)
    if centroids is None:
        out = device_ndarray(_new((nc, k), torch.float32, handle))
        c = cai_wrapper(out)
    else:
        out = centroids
        c = _centroids_out(centroids, nc, k, handle)
    labels = _new((m,), torch.int32, handle) if want_labels else None
    sizes = _new((nc,), torch.int32, handle) if want_labels else None
    need = _lib.lib().b2d_kmeans_balanced_workspace_bytes(m, k, nc)
    if need == 2 ** 64 - 1:
        raise ValueError("invalid extents m=%d, k=%d, n_clusters=%d" % (m, k, nc))
    ws = handle.workspace(need)
    _lib.check(_lib.lib().b2d_kmeans_balanced_fit(handle.stream_ptr, nc, params.n_iters, params.seed & (2 ** 64 - 1),
                                                  x.data, k, m, k, c.data,
                                                  labels.data_ptr() if labels is not None else None,
                                                  sizes.data_ptr() if sizes is not None else None, ws.data_ptr(),
                                                  ws.numel()))
    return out, labels, sizes


@auto_sync_handle
@auto_convert_output
def fit(params, X, n_clusters=None, centroids=None, handle=None):
    """Fits ``n_clusters`` balanced centroids to X (float32 [m, k], C contiguous) and returns them, [n_clusters, k]
    float32 (written into ``centroids`` when given; n_clusters then defaults to its row count)."""
    return _fit(params, X, n_clusters, centroids, False, handle)[0]


@auto_sync_handle
@auto_convert_output
def predict(params, X, centroids, handle=None):
    """int32 [m] labels: the nearest centroid of every row (ties to the smaller index, -1 for a row with NaN)."""
    if params.metric not in ("sqeuclidean", "L2Expanded"):
        raise _lib.LogicError("kmeans_balanced supports the sqeuclidean (L2Expanded) metric only")
    x = _matrix(X, "X")
    m, k = x.shape
    c = _matrix(centroids, "centroids")
    nc = c.shape[0]
    if c.shape[1] != k:
        raise ValueError("centroids must have %d columns, got %d" % (k, c.shape[1]))
    labels = _new((m,), torch.int32, handle)
    inertia = _new((1,), torch.float64, handle)
    ws = _ws(m, k, nc, handle)
    _lib.check(_lib.lib().b2d_kmeans_predict(handle.stream_ptr, x.data, k, None, m, k, c.data, nc, labels.data_ptr(),
                                             inertia.data_ptr(), 1, ws.data_ptr(), ws.numel()))
    return device_ndarray(labels)


@auto_sync_handle
@auto_convert_output
def fit_predict(params, X, n_clusters, handle=None):
    """Returns ``(centroids float32 [n_clusters, k], labels int32 [m], sizes int32 [n_clusters])``: the labels are the
    assignment of the fit's last update (label -1 for a row with a non-finite element) and sizes its cluster sizes, so
    the centroids are ``compute_new_centroids(X, centroids, labels)`` bit for bit."""
    out, labels, sizes = _fit(params, X, n_clusters, None, True, handle)
    return out, device_ndarray(labels), device_ndarray(sizes)
