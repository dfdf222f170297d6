"""DBSCAN -- density-based clustering on the fused epsilon neighbourhood or, for 2-D and 3-D points, on the random ball
cover (cuML's ``DBSCAN(eps, min_samples, metric, max_mbytes_per_batch, algorithm)`` with sklearn.cluster.DBSCAN's
``labels_`` and ``core_sample_indices_``).  Dispatches through the C ABI (include/raft_b200.h: b2d_dbscan_fit and
b2d_dbscan_rbc_fit); the whole fit runs on the device without synchronising."""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from ..distance.distance_type import DistanceType, resolve_metric

DbscanOutput = namedtuple("DbscanOutput", "labels core_sample_indices n_clusters")

METRICS = (DistanceType.L2SqrtExpanded, DistanceType.L2Expanded, DistanceType.CosineExpanded)
# algorithm="rbc": the ball cover's unexpanded distances for "euclidean" / "sqeuclidean"
RBC_METRICS = {DistanceType.L2SqrtExpanded: DistanceType.L2SqrtUnexpanded,
               DistanceType.L2Expanded: DistanceType.L2Unexpanded}


@auto_sync_handle
def dbscan(X, eps, min_samples=5, metric="euclidean", max_mbytes_per_batch=None, algorithm="brute", n_landmarks=None,
           seed=0, handle=None):
    """DBSCAN of the rows of X (float32 [m, d] on the device, rows contiguous, any row pitch >= d, d <= 320).

    metric: "euclidean" (distance <= eps), "sqeuclidean" (squared distance <= eps) or "cosine" (cosine distance <= eps).
    A row is core when at least ``min_samples`` rows, itself included, lie within eps of it.  Clusters are the connected
    components of the core rows, numbered in order of their smallest row; a non-core row within eps of a core row takes
    the smallest such cluster, any other row is noise (-1).  ``max_mbytes_per_batch`` (MiB, default 1024) bounds the
    adjacency bytes formed at once; the result does not depend on it.

    ``algorithm="rbc"`` (d = 2 or 3, euclidean or sqeuclidean) finds the neighbourhoods on a random ball cover of X built
    with ``n_landmarks`` landmarks (default ceil(sqrt(m))) sampled by ``seed``, in O(m) memory; the result depends on
    neither.  It compares the unexpanded distance ``neighbors.ball_cover`` computes, so it can differ from
    ``algorithm="brute"`` (the expanded form) only on pairs whose distance lies within rounding of eps.  It has no
    batches: ``max_mbytes_per_batch`` must stay None.

    Returns ``DbscanOutput(labels, core_sample_indices, n_clusters)``: int32 labels [m] and the core rows in ascending
    order (int32) as torch tensors on the device, and the cluster count as an int (read after the fit).  Raises
    ValueError when X holds NaN or infinity."""
    x = cai_wrapper(X)
    x.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    m, d = x.shape
    if m > 1 and d > 1 and x.strides[1] != 4:
        raise ValueError("X must have contiguous rows")
    ldx = x.strides[0] // 4 if m > 1 else d
    if ldx < d or (m > 1 and x.strides[0] % 4):
        raise ValueError("X must be row-major with a row pitch of at least d elements")
    mt = resolve_metric(metric)
    if mt not in METRICS:
        raise _lib.LogicError("dbscan supports the euclidean, sqeuclidean and cosine metrics, got %r" % (metric,))
    if int(min_samples) < 1:
        raise _lib.LogicError("min_samples must be >= 1, got %r" % (min_samples,))
    if algorithm not in ("brute", "rbc"):
        raise _lib.LogicError("algorithm must be 'brute' or 'rbc', got %r" % (algorithm,))
    rbc = algorithm == "rbc"
    if rbc:
        if mt not in RBC_METRICS:
            raise _lib.LogicError("dbscan(algorithm='rbc') supports the euclidean and sqeuclidean metrics, got %r"
                                  % (metric,))
        if d not in (2, 3):
            raise _lib.LogicError("dbscan(algorithm='rbc') supports d = 2 and d = 3, got d = %d" % d)
        if max_mbytes_per_batch is not None:
            raise _lib.LogicError("dbscan(algorithm='rbc') has no batches: max_mbytes_per_batch must be None")
        nl = 0 if n_landmarks is None else int(n_landmarks)
        if not 0 <= nl <= m:
            raise _lib.LogicError("n_landmarks must be in [0, m] (0 or None: ceil(sqrt(m))), got %r" % (n_landmarks,))
    mb = 0 if max_mbytes_per_batch is None else int(max_mbytes_per_batch * (1 << 20))
    with torch.cuda.stream(handle.torch_stream):
        labels = torch.empty((m,), dtype=torch.int32, device=handle.device)
        core = torch.empty((m,), dtype=torch.int32, device=handle.device)
        ncl = torch.zeros((1,), dtype=torch.int32, device=handle.device)
        if not bool(torch.isfinite(torch.as_tensor(X, device=handle.device)).all()):
            raise ValueError("Input X contains NaN or infinity")
    L = _lib.lib()
    if rbc:
        need = L.b2d_dbscan_rbc_workspace_bytes(m, d, nl)
        ws = handle.workspace(need if need != 2 ** 64 - 1 else 0)
        _lib.check(L.b2d_dbscan_rbc_fit(handle.stream_ptr, int(RBC_METRICS[mt]), x.data, ldx, m, d, float(eps),
                                        int(min_samples), nl, int(seed) & (2 ** 64 - 1), labels.data_ptr(),
                                        core.data_ptr(), ncl.data_ptr(), ws.data_ptr(), ws.numel()))
    else:
        need = L.b2d_dbscan_workspace_bytes(m, d, mb)
        ws = handle.workspace(need if need != 2 ** 64 - 1 else 0)
        _lib.check(L.b2d_dbscan_fit(handle.stream_ptr, int(mt), x.data, ldx, m, d, float(eps), int(min_samples), mb,
                                    labels.data_ptr(), core.data_ptr(), ncl.data_ptr(), ws.data_ptr(), ws.numel()))
    handle.sync()
    n_core = int((core >= 0).sum().item())
    return DbscanOutput(labels, core[:n_core], int(ncl.item()))
