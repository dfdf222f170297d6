"""raft::cluster::single_linkage -- single-linkage clustering on the kNN graph (``LinkageDistance::KNN_GRAPH``) or, for
2-D and 3-D points, exactly over all pairs (``PAIRWISE``) on the random ball cover; the minimum spanning forest of an
edge list, and the exact Euclidean minimum spanning tree of 2-D and 3-D points.  Dispatches through the C ABI
(include/raft_b200.h: b2d_single_linkage, b2d_single_linkage_rbc, b2d_mst, b2d_emst_rbc).  Results are deterministic."""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from ..distance.distance_type import DistanceType, resolve_metric
from .dbscan import RBC_METRICS

LinkageOutput = namedtuple("LinkageOutput", "children deltas sizes labels n_connected_components")
MstOutput = namedtuple("MstOutput", "src dst weights colour")
EmstOutput = namedtuple("EmstOutput", "src dst weights")


def _new(shape, dtype, handle):
    with torch.cuda.stream(handle.torch_stream):
        return torch.empty(shape, dtype=dtype, device=handle.device)


def _rbc_args(X, metric, n_landmarks, fn):
    """the checks of dbscan(algorithm="rbc"): (x, m, d, ldx, unexpanded metric, n_landmarks)"""
    x = cai_wrapper(X)
    x.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    m, d = x.shape
    if m > 1 and d > 1 and x.strides[1] != 4:
        raise ValueError("X must have contiguous rows")
    ldx = x.strides[0] // 4 if m > 1 else d
    if ldx < d or (m > 1 and x.strides[0] % 4):
        raise ValueError("X must be row-major with a row pitch of at least d elements")
    mt = resolve_metric(metric)
    if mt not in RBC_METRICS:
        raise _lib.LogicError("%s supports the euclidean and sqeuclidean metrics, got %r" % (fn, metric))
    if d not in (2, 3):
        raise _lib.LogicError("%s supports d = 2 and d = 3, got d = %d" % (fn, d))
    nl = 0 if n_landmarks is None else int(n_landmarks)
    if not 0 <= nl <= m:
        raise _lib.LogicError("n_landmarks must be in [0, m] (0 or None: ceil(sqrt(m))), got %r" % (n_landmarks,))
    return x, m, d, ldx, RBC_METRICS[mt], nl


@auto_sync_handle
def single_linkage(X, n_clusters, metric="euclidean", c=15, linkage="knn_graph", n_landmarks=None, seed=0, handle=None):
    """Single-linkage clustering of the rows of X (float32 [m, d]).

    ``linkage="knn_graph"`` (X C-contiguous, d <= 320): over the kNN graph with n_nb = min(m, max(2, floor(log2 m) +
    c)) neighbours; the components the graph leaves apart are joined by their nearest rows (connect_components).
    metric: "euclidean" / "l2" (L2SqrtExpanded) or "sqeuclidean" (L2Expanded).

    ``linkage="pairwise"`` (d = 2 or 3, rows contiguous, any row pitch): exactly over all pairs, from the Euclidean
    minimum spanning tree (``emst``), so ``c`` is ignored and ``n_connected_components`` is 1.  The distances are the
    unexpanded ones ``neighbors.ball_cover`` computes ("euclidean": their correctly rounded roots); the result is
    ``scipy.cluster.hierarchy.linkage(method="single")`` on them, up to the order scipy picks among equal heights.
    ``n_landmarks`` (default ceil(sqrt(m))) and ``seed`` shape the ball cover only, never the result.  A non-finite X
    raises LogicError.

    For both, the tree and the merge order are the same for the two metrics, only ``deltas`` differ.

    Returns ``LinkageOutput(children, deltas, sizes, labels, n_connected_components)`` as torch tensors on the device
    (scipy.cluster.hierarchy.linkage's conventions): merge t creates cluster m + t from ``children[t]`` (int32, smaller
    id first) at distance ``deltas[t]`` (float32) with ``sizes[t]`` rows; ``labels`` (int32 [m]) are the clusters after
    the first m - n_clusters merges, numbered in order of their smallest row.  ``n_connected_components`` (int) counts
    the components of the kNN graph.  The call synchronises the handle's stream."""
    if linkage not in ("knn_graph", "pairwise"):
        raise _lib.LogicError("linkage must be 'knn_graph' or 'pairwise', got %r" % (linkage,))
    if linkage == "pairwise":
        x, m, d, ldx, mt, nl = _rbc_args(X, metric, n_landmarks, "single_linkage(linkage='pairwise')")
        L = _lib.lib()
        children = _new((max(m - 1, 0), 2), torch.int32, handle)
        deltas = _new((max(m - 1, 0),), torch.float32, handle)
        sizes = _new((max(m - 1, 0),), torch.int32, handle)
        labels = _new((m,), torch.int32, handle)
        need = L.b2d_single_linkage_rbc_workspace_bytes(m, d, nl)
        ws = handle.workspace(need if need != 2 ** 64 - 1 else 0)
        _lib.check(L.b2d_single_linkage_rbc(handle.stream_ptr, int(mt), x.data, ldx, m, d, nl, int(seed) & (2 ** 64 - 1),
                                            int(n_clusters), children.data_ptr(), deltas.data_ptr(), sizes.data_ptr(),
                                            labels.data_ptr(), ws.data_ptr(), ws.numel()))
        return LinkageOutput(children, deltas, sizes, labels, 1)
    x = cai_wrapper(X)
    x.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if not x.c_contiguous:
        raise _lib.LogicError("X must be C contiguous")
    m, d = x.shape
    mt = resolve_metric(metric)
    if mt not in (DistanceType.L2Expanded, DistanceType.L2SqrtExpanded):
        raise _lib.LogicError("single_linkage supports the euclidean and sqeuclidean metrics, got %r" % (metric,))
    L = _lib.lib()
    children = _new((max(m - 1, 0), 2), torch.int32, handle)
    deltas = _new((max(m - 1, 0),), torch.float32, handle)
    sizes = _new((max(m - 1, 0),), torch.int32, handle)
    labels = _new((m,), torch.int32, handle)
    ncomp = np.zeros(1, np.int32)
    need = L.b2d_single_linkage_workspace_bytes(m, d, int(c))
    ws = handle.workspace(need if need != 2 ** 64 - 1 else 0)
    _lib.check(L.b2d_single_linkage(handle.stream_ptr, int(mt), x.data, d, m, d, int(c), int(n_clusters),
                                    children.data_ptr(), deltas.data_ptr(), sizes.data_ptr(), labels.data_ptr(),
                                    ncomp.ctypes.data, ws.data_ptr(), ws.numel()))
    return LinkageOutput(children, deltas, sizes, labels, int(ncomp[0]))


@auto_sync_handle
def mst(src, dst, weights, n_vertices, handle=None):
    """Minimum spanning forest of the edge list (src[e], dst[e], weights[e]) on ``n_vertices`` vertices (int32
    endpoints, float32 weights, 1-d device arrays), edges ordered by (weight, position e).  Returns
    ``MstOutput(src, dst, weights, colour)``: the forest's edges in that order, as given, and ``colour[v]`` = the smallest
    vertex of v's tree (torch tensors on the device)."""
    n = int(n_vertices)
    arrs = []
    for a, dt, name in ((src, np.int32, "src"), (dst, np.int32, "dst"), (weights, np.float32, "weights")):
        w = cai_wrapper(a)
        w.validate_shape_dtype(expected_dims=1, expected_dtype=dt)
        arrs.append(w)
    e = arrs[0].shape[0]
    if arrs[1].shape[0] != e or arrs[2].shape[0] != e:
        raise ValueError("src, dst and weights must have the same length")
    L = _lib.lib()
    cap = max(n - 1, 1)
    os_, od = _new((cap,), torch.int32, handle), _new((cap,), torch.int32, handle)
    ow, colour = _new((cap,), torch.float32, handle), _new((max(n, 1),), torch.int32, handle)
    count = _new((1,), torch.int32, handle)
    ws = handle.workspace(L.b2d_mst_workspace_bytes(n, e) if n >= 0 else 0)
    _lib.check(L.b2d_mst(handle.stream_ptr, arrs[0].data if e else None, arrs[1].data if e else None,
                         arrs[2].data if e else None, n, e, os_.data_ptr(), od.data_ptr(), ow.data_ptr(),
                         colour.data_ptr(), count.data_ptr(), ws.data_ptr(), ws.numel()))
    handle.sync()
    k = int(count.item())
    return MstOutput(os_[:k], od[:k], ow[:k], colour[:n])


@auto_sync_handle
def emst(X, metric="euclidean", n_landmarks=None, seed=0, handle=None):
    """The exact Euclidean minimum spanning tree of the rows of X (float32 [m, d] on the device, d = 2 or 3, rows
    contiguous, any row pitch), built by Borůvka over a random ball cover of X.  Pair (i, j) weighs the unexpanded squared
    distance ``neighbors.ball_cover`` computes, s; edges are ordered by (s, min(i, j), max(i, j)), so the tree is
    unique.  Returns ``EmstOutput(src, dst, weights)``: the m - 1 edges in that order (int32 rows with src < dst, torch
    tensors on the device) and their weights: s for "sqeuclidean", its correctly rounded root for "euclidean".
    ``n_landmarks`` (default ceil(sqrt(m))) and ``seed`` shape the ball cover only, never the result.  Raises ValueError
    when X holds NaN or infinity."""
    x, m, d, ldx, mt, nl = _rbc_args(X, metric, n_landmarks, "emst")
    if m < 1:
        raise _lib.LogicError("emst needs at least one row")
    src = _new((max(m - 1, 0),), torch.int32, handle)
    dst = _new((max(m - 1, 0),), torch.int32, handle)
    w = _new((max(m - 1, 0),), torch.float32, handle)
    with torch.cuda.stream(handle.torch_stream):
        if not bool(torch.isfinite(torch.as_tensor(X, device=handle.device)).all()):
            raise ValueError("Input X contains NaN or infinity")
    L = _lib.lib()
    need = L.b2d_emst_rbc_workspace_bytes(m, d, nl)
    ws = handle.workspace(need if need != 2 ** 64 - 1 else 0)
    _lib.check(L.b2d_emst_rbc(handle.stream_ptr, int(mt), x.data, ldx, m, d, nl, int(seed) & (2 ** 64 - 1),
                              src.data_ptr(), dst.data_ptr(), w.data_ptr(), ws.data_ptr(), ws.numel()))
    return EmstOutput(src, dst, w)
