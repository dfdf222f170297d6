"""HDBSCAN of 2-D and 3-D points on the random ball cover (sklearn.cluster.HDBSCAN(metric="precomputed") on the ball
cover's pair distances; cuML's HDBSCAN with its ``minimum_spanning_tree_``).  Dispatches through the C ABI
(include/raft_b200.h: b2d_hdbscan_rbc_fit): core distances and the mutual-reachability tree on the device, the tree stages
on the host.  ``hdbscan_model`` also keeps the fitted model, in which ``approximate_predict`` places new points
(b2d_hdbscan_rbc_fit_model, b2d_hdbscan_rbc_approximate_predict)."""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from .single_linkage import EmstOutput, _new, _rbc_args

HdbscanOutput = namedtuple("HdbscanOutput", "labels probabilities n_clusters mst")
HdbscanPrediction = namedtuple("HdbscanPrediction", "labels probabilities neighbors weights")

METHODS = {"eom": 0, "leaf": 1}


@auto_sync_handle
def hdbscan(X, min_cluster_size=5, min_samples=None, cluster_selection_epsilon=0.0, cluster_selection_method="eom",
            allow_single_cluster=False, metric="euclidean", n_landmarks=None, seed=0, handle=None):
    """HDBSCAN of the rows of X (float32 [m, d] on the device, d = 2 or 3, rows contiguous, any row pitch).

    Pair (i, j) is at the unexpanded distance ``neighbors.ball_cover`` computes ("euclidean": the correctly rounded root
    of the squared distance s, "sqeuclidean": s).  The core distance of a row is its ``min_samples``-th smallest distance
    (``min_samples`` defaults to ``min_cluster_size``, 1 <= min_samples <= min(64, m)), the row itself included, and
    pair (i, j) weighs max(core_i, core_j, d(i, j)).  The mutual-reachability tree takes edges in the order (weight, min
    row, max row), so it is unique; the result is sklearn.cluster.HDBSCAN(metric="precomputed", min_cluster_size,
    min_samples, cluster_selection_epsilon, cluster_selection_method, allow_single_cluster) on the matrix of those
    distances when its tree merges in that order (always, when the tree's weights are distinct).  ``n_landmarks``
    (default ceil(sqrt(m))) and ``seed`` shape the ball cover only, never the result.  A non-finite X raises LogicError.

    Returns ``HdbscanOutput(labels, probabilities, n_clusters, mst)``: labels (int32 [m], -1 noise, clusters numbered in
    order of their smallest row) and probabilities (float32 [m]) as torch tensors on the device, the cluster count, and
    the tree as ``EmstOutput(src, dst, weights)``: its m - 1 edges in order, src < dst, at the metric's distance.  The
    call synchronises the handle's stream."""
    return _fit(X, min_cluster_size, min_samples, cluster_selection_epsilon, cluster_selection_method,
                allow_single_cluster, metric, n_landmarks, seed, handle, False)[0]


class HdbscanModel:
    """A fitted HDBSCAN that can place new points (``approximate_predict``): the fit's ``output`` (an
    ``HdbscanOutput``), the device buffer that holds the fit's ball cover, core distances and condensed tree, and the
    extents the buffer was fitted with."""

    def __init__(self, output, buffer, m, d, metric, n_landmarks, min_samples):
        self.output = output
        self.buffer = buffer
        self.m = m
        self.d = d
        self.metric = metric
        self.n_landmarks = n_landmarks
        self.min_samples = min_samples


def _fit(X, min_cluster_size, min_samples, cluster_selection_epsilon, cluster_selection_method, allow_single_cluster,
         metric, n_landmarks, seed, handle, with_model):
    x, m, d, ldx, mt, nl = _rbc_args(X, metric, n_landmarks, "hdbscan")
    mcs = int(min_cluster_size)
    ms = mcs if min_samples is None else int(min_samples)
    if mcs < 2:
        raise _lib.LogicError("min_cluster_size must be at least 2, got %r" % (min_cluster_size,))
    if not 1 <= ms <= min(64, m):
        raise _lib.LogicError("min_samples must be in [1, min(64, m)], got %r" % (ms,))
    eps = float(cluster_selection_epsilon)
    if not 0.0 <= eps < float("inf"):
        raise _lib.LogicError("cluster_selection_epsilon must be finite and non-negative, got %r"
                              % (cluster_selection_epsilon,))
    if cluster_selection_method not in METHODS:
        raise _lib.LogicError("cluster_selection_method must be 'eom' or 'leaf', got %r" % (cluster_selection_method,))
    labels = _new((m,), torch.int32, handle)
    prob = _new((m,), torch.float32, handle)
    src = _new((max(m - 1, 0),), torch.int32, handle)
    dst = _new((max(m - 1, 0),), torch.int32, handle)
    w = _new((max(m - 1, 0),), torch.float32, handle)
    nc = np.zeros(1, np.int32)
    L = _lib.lib()
    need = L.b2d_hdbscan_rbc_workspace_bytes(m, d, nl)
    ws = handle.workspace(need if need != 2 ** 64 - 1 else 0)
    args = (handle.stream_ptr, int(mt), x.data, ldx, m, d, ms, mcs, eps, METHODS[cluster_selection_method],
            int(bool(allow_single_cluster)), nl, int(seed) & (2 ** 64 - 1), labels.data_ptr(), prob.data_ptr(),
            src.data_ptr(), dst.data_ptr(), w.data_ptr(), nc.ctypes.data, ws.data_ptr(), ws.numel())
    model = None
    if with_model:
        size = L.b2d_hdbscan_rbc_model_bytes(m, d, nl)
        model = _new((size if size != 2 ** 64 - 1 else 0,), torch.uint8, handle)
        _lib.check(L.b2d_hdbscan_rbc_fit_model(*args, model.data_ptr() if model.numel() else None))
    else:
        _lib.check(L.b2d_hdbscan_rbc_fit(*args))
    return HdbscanOutput(labels, prob, int(nc[0]), EmstOutput(src, dst, w)), model, (m, d, int(mt), nl, ms)


@auto_sync_handle
def hdbscan_model(X, min_cluster_size=5, min_samples=None, cluster_selection_epsilon=0.0,
                  cluster_selection_method="eom", allow_single_cluster=False, metric="euclidean", n_landmarks=None,
                  seed=0, handle=None):
    """``hdbscan`` with the same arguments, keeping the fitted model for ``approximate_predict``.  Returns an
    ``HdbscanModel`` whose ``output`` is what ``hdbscan`` returns for these arguments, bit for bit.  The model holds its
    own copy of X, so X may change or go afterwards.  The call synchronises the handle's stream."""
    out, buf, (m, d, mt, nl, ms) = _fit(X, min_cluster_size, min_samples, cluster_selection_epsilon,
                                        cluster_selection_method, allow_single_cluster, metric, n_landmarks, seed,
                                        handle, True)
    return HdbscanModel(out, buf, m, d, mt, nl, ms)


@auto_sync_handle
def approximate_predict(model, points, handle=None):
    """Places new points (float32 [q, d] on the device, d the model's, rows contiguous, any row pitch) in a fitted
    ``HdbscanModel``, as the hdbscan package's and cuML's ``approximate_predict`` do, but exactly: a point's core distance
    is its ``min_samples``-th smallest distance to the fitted rows, its neighbour is the first fitted row in the order
    (mutual-reachability weight, distance, row) over all the fitted rows (the hdbscan package looks only at the
    2 min_samples nearest), and the point joins the condensed tree below that neighbour's cluster at
    lambda = min(1 / weight, the neighbour's lambda).  Labels follow the fit's numbering and rule; a fitted row given
    back (on data without duplicate rows) gets its own label and probability.  A point with a non-finite coordinate is
    noise, with neighbour -1 and weight +inf.  The results do not depend on n_landmarks, seed, the order of the points or
    the batching.  include/raft_b200.h, b2d_hdbscan_rbc_approximate_predict, states the contract.

    Returns ``HdbscanPrediction(labels, probabilities, neighbors, weights)``: int32 labels (-1 noise), float32
    probabilities, the int32 neighbour rows and their float32 weights (in the metric's units), as torch tensors on the
    device.  With a handle given, the call only enqueues work on its stream."""
    if not isinstance(model, HdbscanModel):
        raise TypeError("model must be an HdbscanModel (from hdbscan_model), got %s" % type(model).__name__)
    q = cai_wrapper(points)
    q.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    mq, d = q.shape
    if d != model.d:
        raise ValueError("points have %d columns, the model %d" % (d, model.d))
    if mq > 1 and q.strides[1] != 4:
        raise ValueError("points must have contiguous rows")
    ldq = q.strides[0] // 4 if mq > 1 else d
    if ldq < d or (mq > 1 and q.strides[0] % 4):
        raise ValueError("points must be row-major with a row pitch of at least d elements")
    labels = _new((mq,), torch.int32, handle)
    prob = _new((mq,), torch.float32, handle)
    nn = _new((mq,), torch.int32, handle)
    w = _new((mq,), torch.float32, handle)
    _lib.check(_lib.lib().b2d_hdbscan_rbc_approximate_predict(
        handle.stream_ptr, model.buffer.data_ptr(), model.m, model.d, model.metric, model.n_landmarks, model.min_samples,
        q.data, ldq, mq, labels.data_ptr(), prob.data_ptr(), nn.data_ptr(), w.data_ptr()))
    return HdbscanPrediction(labels, prob, nn, w)
