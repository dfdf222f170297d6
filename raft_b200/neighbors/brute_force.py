"""brute_force.knn -- mirror of ``pylibraft.neighbors.brute_force.knn`` (removed upstream together with
the distance package, CHANGELOG.md:59-60; SURVEY.md 8(f2)): exact k nearest neighbours for the L2
metrics and the cosine family, fused -- the m x n distance matrix is never materialised (raft_b200/csrc/expanded_tc.cuh,
EPI_TOPK)."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from ..distance.distance_type import resolve_metric

_METRICS = ("sqeuclidean", "l2", "euclidean", "cosine", "correlation")


@auto_sync_handle
def knn(dataset, queries, k=None, indices=None, distances=None, metric="sqeuclidean", metric_arg=2.0,
        global_id_offset=0, handle=None):
    """Returns ``(distances float32 [n_queries, k], indices int64 [n_queries, k])``: for every query row
    its k nearest rows of ``dataset`` in ascending (distance, index) order.

    dataset [n, d] and queries [m, d]: any C-contiguous float32 ``__cuda_array_interface__`` objects.
    ``indices`` / ``distances``: optional preallocated outputs (k is then read from their shape).
    metric: "sqeuclidean" (squared), "euclidean" / "l2", "cosine" or "correlation" (pylibraft's names).
    Rows of ``dataset`` whose distance is NaN (a NaN element, a zero-norm row under cosine) are never returned; a
    slot without a candidate (a NaN or zero-norm query) gets index -1 and distance +inf, ``global_id_offset`` or not."""
    if metric not in _METRICS:
        raise ValueError("metric %s is not supported by the fused kNN (L2 metrics, cosine, correlation)" % metric)
    d_cai, q_cai = cai_wrapper(dataset), cai_wrapper(queries)
    d_cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    q_cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if d_cai.shape[1] != q_cai.shape[1]:
        raise ValueError("Inputs must have same number of columns. a=%s, b=%s" % (d_cai.shape[1], q_cai.shape[1]))
    if not (d_cai.c_contiguous and q_cai.c_contiguous):
        raise ValueError("Inputs must be C contiguous")
    n, dim = d_cai.shape
    m = q_cai.shape[0]
    if k is None:
        if indices is not None:
            k = cai_wrapper(indices).shape[1]
        elif distances is not None:
            k = cai_wrapper(distances).shape[1]
        else:
            raise ValueError("Argument k must be specified if both indices and distances arg is None")
    k = int(k)
    with torch.cuda.stream(handle.torch_stream):
        idx = torch.empty((m, k), dtype=torch.int64, device=handle.device)
        dist = torch.empty((m, k), dtype=torch.float32, device=handle.device)
    L = _lib.lib()
    need = L.b2d_knn_l2_workspace_bytes(m, n, dim, k)
    if need == 2 ** 64 - 1:
        raise _lib.LogicError("k must be between 1 and 64")
    ws = handle.workspace(need)
    _lib.check(L.b2d_knn(handle.stream_ptr, idx.data_ptr(), dist.data_ptr(), int(resolve_metric(metric)), q_cai.data, dim,
                         d_cai.data, dim, m, n, dim, k, ws.data_ptr(), ws.numel()))
    if global_id_offset:   # a slot without a candidate keeps index -1
        with torch.cuda.stream(handle.torch_stream):
            idx.copy_(torch.where(idx >= 0, idx + int(global_id_offset), idx))
    for out, res in ((indices, idx), (distances, dist)):
        if out is not None:
            o = cai_wrapper(out)
            if tuple(o.shape) != (m, k):
                raise ValueError("output shape must be (n_queries, k)")
            with torch.cuda.stream(handle.torch_stream):
                torch.as_tensor(out, device=handle.device).copy_(res)
    return (distances if distances is not None else dist), (indices if indices is not None else idx)
