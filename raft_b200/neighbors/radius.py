"""radius_neighbors -- every dataset row within a radius of each query row, as CSR with distances (the answer of
``sklearn.neighbors.NearestNeighbors.radius_neighbors(sort_results=True)``), fused into the tensor-core distance kernel so
the m x n distance matrix is never written (raft_b200/csrc/radius.cu, expanded_tc.cuh EPI_RADIUS).  A project API: pylibraft
never had this entry point, so there is no pylibraft alias."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from ..distance.distance_type import resolve_metric

_METRICS = ("sqeuclidean", "l2", "euclidean", "cosine", "correlation")
MAX_K = 320          # the whole distance of a pair is formed at once
MAX_NNZ = 2 ** 31 - 1   # pairs per call (the segmented sort counts items in an int)


@auto_sync_handle
def radius_neighbors(dataset, queries, radius, metric="sqeuclidean", handle=None):
    """Returns ``(indptr, indices, distances)``: CSR rows, one per query row, holding the rows j of ``dataset`` with
    ``d(q_i, x_j) <= radius``.

    dataset [n, d] and queries [m, d]: C-contiguous float32 ``__cuda_array_interface__`` objects, d <= 320.
    metric: "sqeuclidean" (``radius`` is then a squared distance), "euclidean" / "l2", "cosine" or "correlation".
    d is bit for bit the float32 value ``pairwise_distance(queries, dataset, metric)`` returns, including its rule that a
    row paired with itself is at 0 under the L2 metrics when ``queries`` is ``dataset`` (a copy gets no such rule).
    A NaN distance (NaN element, zero-norm row under cosine, constant row under correlation) is never in the result; a NaN
    or negative radius gives no pairs and ``radius = inf`` every non-NaN pair.

    Outputs (torch tensors on the handle's device): ``indptr`` int64 [m + 1], ``indices`` int64 [nnz] and ``distances``
    float32 [nnz].  Each row is sorted by (distance, index): equal distances by ascending index, -0.0 before +0.0, as in
    ``brute_force.knn``; the result is the same bytes on every call.  Two passes over the pairs: the first counts them per
    row, then ``indptr[m]`` is read on the host -- the call's one synchronisation, as with ``torch.nonzero`` -- and the
    second writes them.  At most 2^31 - 1 pairs per call (LogicError otherwise: split the queries).

    To scipy or torch sparse matrices of shape (m, n)::

        indptr, indices, distances = radius_neighbors(x, q, r)
        scipy.sparse.csr_matrix((distances.cpu().numpy(), indices.cpu().numpy(), indptr.cpu().numpy()), shape=(m, n))
        torch.sparse_csr_tensor(indptr, indices, distances, size=(m, n))

    (A sparse matrix drops nothing, but a zero distance reads as an absent entry in dense views.)"""
    if metric not in _METRICS:
        raise ValueError("metric %s is not supported by radius_neighbors (L2 metrics, cosine, correlation)" % metric)
    d_cai, q_cai = cai_wrapper(dataset), cai_wrapper(queries)
    d_cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    q_cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if d_cai.shape[1] != q_cai.shape[1]:
        raise ValueError("Inputs must have same number of columns. a=%s, b=%s" % (d_cai.shape[1], q_cai.shape[1]))
    if not (d_cai.c_contiguous and q_cai.c_contiguous):
        raise ValueError("Inputs must be C contiguous")
    n, dim = d_cai.shape
    m = q_cai.shape[0]
    if dim > MAX_K:
        raise _lib.LogicError("radius_neighbors supports d <= %d, got d = %d" % (MAX_K, dim))
    metric_id = int(resolve_metric(metric))
    radius = float(radius)
    L = _lib.lib()
    with torch.cuda.stream(handle.torch_stream):
        indptr = torch.empty(m + 1, dtype=torch.int64, device=handle.device)
    ws = handle.workspace(L.b2d_radius_neighbors_workspace_bytes(m, n, dim, 0))
    _lib.check(L.b2d_radius_neighbors_count(handle.stream_ptr, indptr.data_ptr(), metric_id, q_cai.data, dim, d_cai.data,
                                            dim, m, n, dim, radius, ws.data_ptr(), ws.numel()))
    with torch.cuda.stream(handle.torch_stream):
        nnz = int(indptr[m].item())   # the one host synchronisation
    if nnz > MAX_NNZ:
        raise _lib.LogicError("radius_neighbors: %d pairs exceed %d per call: split the queries into smaller batches"
                              % (nnz, MAX_NNZ))
    with torch.cuda.stream(handle.torch_stream):
        indices = torch.empty(nnz, dtype=torch.int64, device=handle.device)
        distances = torch.empty(nnz, dtype=torch.float32, device=handle.device)
    if nnz:
        ws = handle.workspace(L.b2d_radius_neighbors_workspace_bytes(m, n, dim, nnz))
        _lib.check(L.b2d_radius_neighbors_fill(handle.stream_ptr, indptr.data_ptr(), nnz, indices.data_ptr(),
                                               distances.data_ptr(), metric_id, q_cai.data, dim, d_cai.data, dim, m, n, dim,
                                               radius, ws.data_ptr(), ws.numel()))
    return indptr, indices, distances
