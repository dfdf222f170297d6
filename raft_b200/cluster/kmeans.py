"""raft::cluster::kmeans -- Lloyd's k-means on the exact fused L2 arg-min, mirror of the historical
``pylibraft.cluster.kmeans`` ([RECALLED]: removed with ``distance/``, CHANGELOG.md:59).  Dispatches through the C ABI
(include/raft_b200.h: b2d_kmeans_*).  A fit runs its whole loop on the device; results are bit-identical from run to
run."""
from __future__ import annotations

import math
from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..common import auto_convert_output, auto_sync_handle, cai_wrapper, device_ndarray

FitOutput = namedtuple("FitOutput", "centroids inertia n_iter")

INIT_METHODS = {
    "KMeansPlusPlus": _lib.B2D_KMEANS_INIT_PLUS_PLUS,
    "Random": _lib.B2D_KMEANS_INIT_RANDOM,
    "Array": _lib.B2D_KMEANS_INIT_ARRAY,
}


class KMeansParams:
    """Parameters of a fit ([RECALLED] pylibraft.cluster.kmeans.KMeansParams).  Only ``metric="sqeuclidean"`` is
    supported (anything else raises LogicError).  ``oversampling_factor``: None or 0 keeps greedy k-means++; a positive
    value with ``init_method="KMeansPlusPlus"`` seeds with k-means|| (see ``init_scalable``) instead; a negative or
    non-finite value raises ValueError.  ``batch_samples``, ``batch_centroids`` and ``verbosity`` are accepted for
    signature compatibility and have no effect: the assignment is never batched."""

    def __init__(self, n_clusters=None, max_iter=300, tol=1e-4, verbosity=None, seed=0, metric="sqeuclidean",
                 init_method="KMeansPlusPlus", n_init=1, oversampling_factor=None, batch_samples=None,
                 batch_centroids=None, inertia_check=False):
        if metric not in ("sqeuclidean", "L2Expanded"):
            raise _lib.LogicError("kmeans supports the sqeuclidean (L2Expanded) metric only, got %r" % (metric,))
        if init_method not in INIT_METHODS:
            raise ValueError("init_method must be one of %s, got %r" % (sorted(INIT_METHODS), init_method))
        self.n_clusters = None if n_clusters is None else int(n_clusters)
        self.max_iter = int(max_iter)
        self.tol = float(tol)
        self.verbosity = verbosity
        self.seed = int(seed)
        self.metric = metric
        self.init_method = init_method
        self.n_init = int(n_init)
        if oversampling_factor is not None:
            oversampling_factor = float(oversampling_factor)
            if not math.isfinite(oversampling_factor) or oversampling_factor < 0:
                raise ValueError("oversampling_factor must be None or finite and >= 0, got %r" % (oversampling_factor,))
        self.oversampling_factor = oversampling_factor
        self.batch_samples = batch_samples
        self.batch_centroids = batch_centroids
        self.inertia_check = bool(inertia_check)


def _matrix(X, name):
    a = cai_wrapper(X)
    a.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if not a.c_contiguous:
        raise _lib.LogicError("%s must be C contiguous" % name)
    return a


def _vector(v, n, dtype, name):
    if v is None:
        return None
    a = cai_wrapper(v)
    a.validate_shape_dtype(expected_dims=1, expected_dtype=dtype)
    if a.shape[0] != n:
        raise ValueError("%s must have shape (%d,), got %s" % (name, n, a.shape))
    return a


def _new(shape, dtype, handle):
    with torch.cuda.stream(handle.torch_stream):
        return torch.empty(shape, dtype=dtype, device=handle.device)


def _centroids_out(centroids, nc, k, handle):
    c = _matrix(centroids, "centroids")
    if c.shape != (nc, k):
        raise ValueError("centroids must have shape %s, got %s" % ((nc, k), c.shape))
    return c


def _ws(m, k, nc, handle):
    return handle.workspace(_lib.lib().b2d_kmeans_workspace_bytes(m, k, nc))


def _ws_scalable(m, k, nc, f, handle):
    need = _lib.lib().b2d_kmeans_scalable_workspace_bytes(m, k, nc, f)
    if need == 2 ** 64 - 1:
        raise _lib.LogicError("k-means|| needs a finite oversampling_factor > 0 and fewer than 2^31 candidates")
    return handle.workspace(need)


@auto_sync_handle
def fit(params, X, centroids=None, sample_weights=None, handle=None):
    """Returns ``FitOutput(centroids, inertia, n_iter)``.  ``centroids``: [n_clusters, k] float32, the initial
    centroids for ``init_method="Array"`` (required then) and the output in every case (written in place when given;
    by default a new ``device_ndarray``).  ``sample_weights``: optional float32 [m], scaled to sum to m.  inertia is
    sum_i w_i min_j ||x_i - c_j||^2 for the returned centroids (a Python float), n_iter the iterations that ran."""
    x = _matrix(X, "X")
    m, k = x.shape
    nc = params.n_clusters
    if centroids is not None and nc is None:
        nc = cai_wrapper(centroids).shape[0]
    if nc is None:
        raise ValueError("n_clusters must be set")
    if params.init_method == "Array" and centroids is None:
        raise ValueError("init_method='Array' needs centroids")
    if centroids is None:
        out = device_ndarray(_new((nc, k), torch.float32, handle))
        c = cai_wrapper(out)
    else:
        out = centroids
        c = _centroids_out(centroids, nc, k, handle)
    w = _vector(sample_weights, m, np.float32, "sample_weights")
    inertia = _new((1,), torch.float64, handle)
    n_iter = _new((1,), torch.int32, handle)
    seed = params.seed & (2 ** 64 - 1)
    f = params.oversampling_factor
    if params.init_method == "KMeansPlusPlus" and f:   # k-means|| seeding
        ws = _ws_scalable(m, k, nc, f, handle)
        _lib.check(_lib.lib().b2d_kmeans_fit_scalable(handle.stream_ptr, nc, params.max_iter, params.tol, f, params.n_init,
                                                      seed, 1 if params.inertia_check else 0, x.data, k,
                                                      w.data if w else None, m, k, c.data, inertia.data_ptr(),
                                                      n_iter.data_ptr(), ws.data_ptr(), ws.numel()))
    else:
        ws = _ws(m, k, nc, handle)
        _lib.check(_lib.lib().b2d_kmeans_fit(handle.stream_ptr, nc, params.max_iter, params.tol,
                                             INIT_METHODS[params.init_method], params.n_init, seed,
                                             1 if params.inertia_check else 0, x.data, k, w.data if w else None, m, k,
                                             c.data, inertia.data_ptr(), n_iter.data_ptr(), ws.data_ptr(), ws.numel()))
    handle.sync()
    return FitOutput(out, float(inertia.item()), int(n_iter.item()))


@auto_sync_handle
@auto_convert_output
def predict(params, X, centroids, sample_weights=None, handle=None, normalize_weight=True):
    """Returns ``(labels int32 [m], inertia float)``: the nearest centroid of every row (ties to the smaller index, -1
    for a row with NaN distances) and sum_i w_i min_j ||x_i - c_j||^2 (weights scaled to sum to m)."""
    x = _matrix(X, "X")
    m, k = x.shape
    c = _matrix(centroids, "centroids")
    nc = c.shape[0]
    if c.shape[1] != k:
        raise ValueError("centroids must have %d columns, got %d" % (k, c.shape[1]))
    w = _vector(sample_weights, m, np.float32, "sample_weights")
    labels = _new((m,), torch.int32, handle)
    inertia = _new((1,), torch.float64, handle)
    ws = _ws(m, k, nc, handle)
    _lib.check(_lib.lib().b2d_kmeans_predict(handle.stream_ptr, x.data, k, w.data if w else None, m, k, c.data, nc,
                                             labels.data_ptr(), inertia.data_ptr(), 1 if normalize_weight else 0,
                                             ws.data_ptr(), ws.numel()))
    handle.sync()
    return device_ndarray(labels), float(inertia.item())


@auto_sync_handle
def cluster_cost(X, centroids, handle=None):
    """sum_i min_j ||x_i - c_j||^2 (a Python float)."""
    return predict(KMeansParams(n_clusters=cai_wrapper(centroids).shape[0]), X, centroids, handle=handle)[1]


@auto_sync_handle
@auto_convert_output
def compute_new_centroids(X, centroids, labels, new_centroids, sample_weights=None, weight_per_cluster=None,
                          handle=None):
    """One update step: new_centroids[j] = sum_{labels_i = j} w_i x_i / sum w_i (fp64 sums rounded once to float32;
    a cluster of zero weight keeps ``centroids[j]``; labels outside [0, n_clusters) are skipped).  The weights are
    used as given.  ``weight_per_cluster``: optional float32 [n_clusters] output of the weight sums.  Returns
    new_centroids."""
    x = _matrix(X, "X")
    m, k = x.shape
    c = _matrix(centroids, "centroids")
    nc = c.shape[0]
    if c.shape[1] != k:
        raise ValueError("centroids must have %d columns, got %d" % (k, c.shape[1]))
    nco = _centroids_out(new_centroids, nc, k, handle)
    lab = _vector(labels, m, np.int32, "labels")
    w = _vector(sample_weights, m, np.float32, "sample_weights")
    wpc = _vector(weight_per_cluster, nc, np.float32, "weight_per_cluster")
    ws = _ws(m, k, nc, handle)
    _lib.check(_lib.lib().b2d_kmeans_update_centroids(handle.stream_ptr, x.data, k, w.data if w else None, lab.data, m, k,
                                                      c.data, nc, nco.data, wpc.data if wpc else None, ws.data_ptr(),
                                                      ws.numel()))
    return new_centroids


@auto_sync_handle
@auto_convert_output
def init_plus_plus(X, n_clusters=None, seed=None, handle=None, centroids=None):
    """Greedy k-means++ seeding: [n_clusters, k] float32 rows of X (written into ``centroids`` when given)."""
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
    ws = _ws(m, k, nc, handle)
    _lib.check(_lib.lib().b2d_kmeans_init_plus_plus(handle.stream_ptr, x.data, k, None, m, k, nc,
                                                    (0 if seed is None else int(seed)) & (2 ** 64 - 1), c.data,
                                                    ws.data_ptr(), ws.numel()))
    return out


@auto_sync_handle
@auto_convert_output
def init_scalable(X, n_clusters=None, oversampling_factor=2.0, seed=None, sample_weights=None, centroids=None,
                  return_candidates=False, handle=None):
    """k-means|| seeding (include/raft_b200.h: b2d_kmeans_init_scalable): 1 + 8L candidate rows drawn in 9 rounds
    (L = min(m, max(ceil(oversampling_factor * n_clusters), ceil((n_clusters - 1) / 8)))), weighted by the weights of
    the rows nearest to them, reclustered into [n_clusters, k] float32 centroids (written into ``centroids`` when
    given).  ``sample_weights``: optional float32 [m], used as given.  With ``return_candidates`` returns
    ``(centroids, candidate_rows int32 [C], candidate_weights float32 [C])``."""
    x = _matrix(X, "X")
    m, k = x.shape
    if n_clusters is None:
        if centroids is None:
            raise ValueError("n_clusters or centroids must be given")
        n_clusters = cai_wrapper(centroids).shape[0]
    nc = int(n_clusters)
    f = float(oversampling_factor)
    if not math.isfinite(f) or f <= 0:
        raise ValueError("oversampling_factor must be finite and > 0, got %r" % (oversampling_factor,))
    if centroids is None:
        out = device_ndarray(_new((nc, k), torch.float32, handle))
        c = cai_wrapper(out)
    else:
        out = centroids
        c = _centroids_out(centroids, nc, k, handle)
    w = _vector(sample_weights, m, np.float32, "sample_weights")
    ws = _ws_scalable(m, k, nc, f, handle)
    n_cand = 1 + 8 * min(m, max(math.ceil(f * nc), math.ceil((nc - 1) / 8)))
    rows = _new((n_cand,), torch.int32, handle) if return_candidates else None
    wts = _new((n_cand,), torch.float32, handle) if return_candidates else None
    _lib.check(_lib.lib().b2d_kmeans_init_scalable(handle.stream_ptr, x.data, k, w.data if w else None, m, k, nc, f,
                                                   (0 if seed is None else int(seed)) & (2 ** 64 - 1), c.data,
                                                   rows.data_ptr() if rows is not None else None,
                                                   wts.data_ptr() if wts is not None else None, ws.data_ptr(),
                                                   ws.numel()))
    if return_candidates:
        return out, device_ndarray(rows), device_ndarray(wts)
    return out
