"""HDBSCAN of 2-D and 3-D points on the random ball cover (sklearn.cluster.HDBSCAN(metric="precomputed") on the ball
cover's pair distances; cuML's HDBSCAN with its ``minimum_spanning_tree_``).  Dispatches through the C ABI
(include/raft_b200.h: b2d_hdbscan_rbc_fit): core distances and the mutual-reachability tree on the device, the tree stages
on the host."""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle
from .single_linkage import EmstOutput, _new, _rbc_args

HdbscanOutput = namedtuple("HdbscanOutput", "labels probabilities n_clusters mst")

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
    _lib.check(L.b2d_hdbscan_rbc_fit(handle.stream_ptr, int(mt), x.data, ldx, m, d, ms, mcs, eps,
                                     METHODS[cluster_selection_method], int(bool(allow_single_cluster)), nl,
                                     int(seed) & (2 ** 64 - 1), labels.data_ptr(), prob.data_ptr(), src.data_ptr(),
                                     dst.data_ptr(), w.data_ptr(), nc.ctypes.data, ws.data_ptr(), ws.numel()))
    return HdbscanOutput(labels, prob, int(nc[0]), EmstOutput(src, dst, w))
