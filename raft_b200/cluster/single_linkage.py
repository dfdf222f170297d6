"""raft::cluster::single_linkage with ``LinkageDistance::KNN_GRAPH`` -- single-linkage clustering on the kNN graph, and
the minimum spanning forest of an edge list it is built on.  Dispatches through the C ABI (include/raft_b200.h:
b2d_single_linkage, b2d_mst).  Results are deterministic: the edges are ordered by (squared weight, position)."""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from ..distance.distance_type import DistanceType, resolve_metric

LinkageOutput = namedtuple("LinkageOutput", "children deltas sizes labels n_connected_components")
MstOutput = namedtuple("MstOutput", "src dst weights colour")


def _new(shape, dtype, handle):
    with torch.cuda.stream(handle.torch_stream):
        return torch.empty(shape, dtype=dtype, device=handle.device)


@auto_sync_handle
def single_linkage(X, n_clusters, metric="euclidean", c=15, handle=None):
    """Single-linkage clustering of the rows of X (float32 [m, d], C-contiguous, d <= 320) over its kNN graph with
    n_nb = min(m, max(2, floor(log2 m) + c)) neighbours; the components the graph leaves apart are joined by their
    nearest rows (connect_components).  metric: "euclidean" / "l2" (L2SqrtExpanded) or "sqeuclidean" (L2Expanded); the
    tree and the merge order are the same for both, only ``deltas`` differ.

    Returns ``LinkageOutput(children, deltas, sizes, labels, n_connected_components)`` as torch tensors on the device
    (scipy.cluster.hierarchy.linkage's conventions): merge t creates cluster m + t from ``children[t]`` (int32, smaller
    id first) at distance ``deltas[t]`` (float32) with ``sizes[t]`` rows; ``labels`` (int32 [m]) are the clusters after
    the first m - n_clusters merges, numbered in order of their smallest row.  ``n_connected_components`` (int) counts
    the components of the kNN graph.  The call synchronises the handle's stream."""
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
