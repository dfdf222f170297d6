"""ball_cover -- the random ball cover: exact kNN and epsilon-neighbourhood queries for 2-D and 3-D points
(``raft::neighbors::ball_cover`` before the move to cuVS; raft_b200/csrc/ball_cover.cu).  A project API like
``radius_neighbors``: the brute-force entry points do all m x n pairs, this one prunes whole balls of points by the
triangle inequality, exactly.

Distances are the UNEXPANDED ones, fixed bit for bit: ``s = ((q0-p0)^2 + (q1-p1)^2) + (q2-p2)^2`` in float32 with every
operation rounded separately; "sqeuclidean" is s and "euclidean" is the correctly rounded sqrt(s).  ``brute_force.knn``
computes the expanded form, so its distances can differ in the last bits and near-ties can come in another order.
Neighbours are ordered by (distance, index); a pair at a NaN distance is never a neighbour.  The answers do not depend on
``seed`` or ``n_landmarks``: those only change how fast they come."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from ..distance.distance_type import DistanceType

_METRICS = {"sqeuclidean": DistanceType.L2Unexpanded, "euclidean": DistanceType.L2SqrtUnexpanded}
SIZE_MAX = 2 ** 64 - 1
MAX_NNZ = 2 ** 31 - 1   # pairs per eps_nn call


class BallCoverIndex:
    """A built ball cover: the device buffer (its own copy of the points, grouped by ball), n, d, the metric id and the
    number of landmarks.  ``dataset`` is kept for ``all_knn_query``."""

    def __init__(self, buffer, dataset, n, d, metric, n_landmarks):
        self.buffer = buffer
        self.dataset = dataset
        self.n = n
        self.d = d
        self.metric = metric
        self.n_landmarks = n_landmarks


def _points(a, name):
    cai = cai_wrapper(a)
    cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if not cai.c_contiguous:
        raise ValueError("%s must be C contiguous" % name)
    return cai


@auto_sync_handle
def build_index(dataset, metric="euclidean", n_landmarks=None, seed=0, handle=None):
    """Builds a ball cover of ``dataset`` [n, d] (C-contiguous float32 CUDA array, d = 2 or 3).

    metric: "euclidean" or "sqeuclidean" (the unexpanded values above).  n_landmarks: the number of balls, in [1, n];
    None for ceil(sqrt(n)).  Landmarks are a uniform sample of the rows drawn from ``seed``."""
    if metric not in _METRICS:
        raise ValueError("metric %s is not supported by ball_cover (euclidean, sqeuclidean)" % metric)
    cai = _points(dataset, "dataset")
    n, d = cai.shape
    nl = 0 if n_landmarks is None else int(n_landmarks)
    L = _lib.lib()
    size = L.b2d_ball_cover_index_bytes(n, d, nl)
    if size == SIZE_MAX:   # invalid extents: the build says which
        _lib.check(L.b2d_ball_cover_build(handle.stream_ptr, None, cai.data, d, n, d, int(_METRICS[metric]), nl, 0, None, 0))
    with torch.cuda.stream(handle.torch_stream):
        buf = torch.empty(size, dtype=torch.uint8, device=handle.device)
    ws = handle.workspace(L.b2d_ball_cover_build_workspace_bytes(n, d, nl))
    _lib.check(L.b2d_ball_cover_build(handle.stream_ptr, buf.data_ptr(), cai.data, d, n, d, int(_METRICS[metric]), nl,
                                      int(seed) % 2 ** 64, ws.data_ptr(), ws.numel()))
    return BallCoverIndex(buf, dataset, n, d, int(_METRICS[metric]), nl)


@auto_sync_handle
def knn_query(index, queries, k, handle=None):
    """Returns ``(distances float32 [m, k], indices int64 [m, k])``: the k nearest rows of the index's dataset for every
    row of ``queries`` [m, d], in ascending (distance, index) order, as ``brute_force.knn`` returns them.  1 <= k <=
    min(64, n).  A slot without a comparable row (a NaN query) has index -1 and distance +inf."""
    q = _points(queries, "queries")
    if q.shape[1] != index.d:
        raise ValueError("queries have %d columns, the index %d" % (q.shape[1], index.d))
    m, k = q.shape[0], int(k)
    with torch.cuda.stream(handle.torch_stream):
        idx = torch.empty((m, k), dtype=torch.int64, device=handle.device)
        dist = torch.empty((m, k), dtype=torch.float32, device=handle.device)
    L = _lib.lib()
    _lib.check(L.b2d_ball_cover_knn(handle.stream_ptr, idx.data_ptr(), dist.data_ptr(), index.buffer.data_ptr(), index.n,
                                    index.d, index.metric, index.n_landmarks, q.data, index.d, m, k))
    return dist, idx


def all_knn_query(index, k, handle=None):
    """``knn_query`` of the index's own dataset: every row finds itself at distance 0 (ties by index)."""
    return knn_query(index, index.dataset, k, handle=handle)


@auto_sync_handle
def eps_nn(index, queries, eps, handle=None):
    """Returns ``(indptr, indices, distances)``: CSR rows, one per query row, of the dataset rows at distance <= eps,
    each row in (distance, index) order -- the answer of ``radius_neighbors`` on the unexpanded distances.  Under
    "sqeuclidean" eps is a squared distance.  A NaN or negative eps gives no pairs.  One host synchronisation, to read
    the number of pairs between the count and the fill pass; at most 2^31 - 1 pairs per call."""
    q = _points(queries, "queries")
    if q.shape[1] != index.d:
        raise ValueError("queries have %d columns, the index %d" % (q.shape[1], index.d))
    m, eps = q.shape[0], float(eps)
    L = _lib.lib()
    args = (index.buffer.data_ptr(), index.n, index.d, index.metric, index.n_landmarks, q.data, index.d, m, eps)
    with torch.cuda.stream(handle.torch_stream):
        indptr = torch.empty(m + 1, dtype=torch.int64, device=handle.device)
    ws = handle.workspace(L.b2d_ball_cover_eps_workspace_bytes(m, 0))
    _lib.check(L.b2d_ball_cover_eps_count(handle.stream_ptr, indptr.data_ptr(), *args, ws.data_ptr(), ws.numel()))
    with torch.cuda.stream(handle.torch_stream):
        nnz = int(indptr[m].item())   # the one host synchronisation
    if nnz > MAX_NNZ:
        raise _lib.LogicError("eps_nn: %d pairs exceed %d per call: split the queries into smaller batches"
                              % (nnz, MAX_NNZ))
    with torch.cuda.stream(handle.torch_stream):
        indices = torch.empty(nnz, dtype=torch.int64, device=handle.device)
        distances = torch.empty(nnz, dtype=torch.float32, device=handle.device)
    if nnz:
        ws = handle.workspace(L.b2d_ball_cover_eps_workspace_bytes(m, nnz))
        _lib.check(L.b2d_ball_cover_eps_fill(handle.stream_ptr, indptr.data_ptr(), nnz, indices.data_ptr(),
                                             distances.data_ptr(), *args, ws.data_ptr(), ws.numel()))
    return indptr, indices, distances
