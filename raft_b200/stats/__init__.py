"""Callers of the distance path (SURVEY.md 8(f3)): ``silhouette_score`` on the raft_b200 engine -- the
role of ``raft::stats::silhouette_score`` (cpp/include/raft/stats/silhouette_score.cuh), whose call into
``raft::distance::pairwise_distance`` is dangling in the reference snapshot
(cpp/include/raft/stats/detail/silhouette_score.cuh:205-206)."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from ..distance.distance_type import resolve_metric


@auto_sync_handle
def silhouette_score(X, labels, n_labels=None, metric="sqeuclidean_unexpanded", p=2.0, chunk=0, return_samples=False,
                     handle=None):
    """Mean silhouette coefficient of the samples X [n, d] (float32, C-contiguous, on the device) under the
    clustering ``labels`` (int32 in [0, n_labels)).  ``metric`` takes the names of ``pairwise_distance``;
    the default is the reference's (DistanceType::L2Unexpanded, i.e. squared Euclidean) -- pass
    "euclidean" for scikit-learn's default.  ``chunk``: rows of the distance matrix alive at a time
    (0: about 1 GiB).  Returns a float, or (float, per-sample scores [n]) with ``return_samples``."""
    x_cai, l_cai = cai_wrapper(X), cai_wrapper(labels)
    x_cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    l_cai.validate_shape_dtype(expected_dims=1, expected_dtype=np.int32)
    if not x_cai.c_contiguous:
        raise ValueError("Inputs must be C contiguous")
    n, d = x_cai.shape
    if l_cai.shape[0] != n:
        raise ValueError("labels must have one entry per sample")
    if n_labels is None:
        n_labels = int(torch.as_tensor(labels, device=handle.device).max().item()) + 1
    mt = int(resolve_metric(metric))
    L = _lib.lib()
    need = L.b2d_silhouette_score_workspace_bytes(n, d, int(n_labels), mt, int(chunk))
    if need == 2 ** 64 - 1:
        raise _lib.LogicError("metric %s is not supported" % metric)
    ws = handle.workspace(need)
    with torch.cuda.stream(handle.torch_stream):
        score = torch.empty(1, dtype=torch.float32, device=handle.device)
        per = torch.empty(n, dtype=torch.float32, device=handle.device) if return_samples else None
    _lib.check(L.b2d_silhouette_score(handle.stream_ptr, score.data_ptr(), per.data_ptr() if per is not None else None,
                                      x_cai.data, d, l_cai.data, n, d, int(n_labels), mt, float(p), int(chunk),
                                      ws.data_ptr(), ws.numel()))
    handle.sync()
    val = float(score.item())
    if val != val:
        # the C ABI validates labels on the device and poisons the score instead of synchronising; this wrapper
        # returns a host float (it has synchronised already), so it can turn that into the reference's error
        lt = torch.as_tensor(labels, device=handle.device)
        if int(lt.min().item()) < 0 or int(lt.max().item()) >= int(n_labels):
            raise _lib.LogicError("labels must lie in [0, n_labels)")
        if int(torch.unique(lt).numel()) < 2:
            raise _lib.LogicError("silhouette score is not defined for fewer than 2 non-empty clusters")
    return (val, per) if return_samples else val


@auto_sync_handle
def trustworthiness_score(X, X_embedded, n_neighbors=5, metric="euclidean", batch_size=0, handle=None):
    """Trustworthiness of the embedding ``X_embedded`` [n, d] of ``X`` [n, m] (both float32, C-contiguous, on
    the device): 1 - 2 / (n k (2n - 3k - 1)) * sum over samples i and their k embedded-space neighbours j
    of max(0, r(i, j) - k), r = rank of j among the original-space neighbours of i
    (raft::stats::trustworthiness_score, cpp/include/raft/stats/trustworthiness_score.cuh:29-41; same
    definition as sklearn.manifold.trustworthiness).  ``metric``: original-space metric (any name of
    ``pairwise_distance`` from the L2 / cosine families); the embedded-space neighbours use the same metric, as in the reference.  ``batch_size``: rows of
    the original-space distance matrix alive at a time (0: about 1 GiB).  Returns a float."""
    import ctypes
    x_cai, e_cai = cai_wrapper(X), cai_wrapper(X_embedded)
    x_cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    e_cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if not (x_cai.c_contiguous and e_cai.c_contiguous):
        raise ValueError("Inputs must be C contiguous")
    n, m = x_cai.shape
    if e_cai.shape[0] != n:
        raise ValueError("Size mismatch between X and X_embedded")
    d = e_cai.shape[1]
    mt = int(resolve_metric(metric))
    L = _lib.lib()
    need = L.b2d_trustworthiness_score_workspace_bytes(n, m, d, int(n_neighbors), mt, int(batch_size))
    if need == 2 ** 64 - 1:
        raise _lib.LogicError("n_neighbors must be in [1, 63] and the metric one of pairwise_distance's")
    ws = handle.workspace(need)
    with torch.cuda.stream(handle.torch_stream):
        out = torch.empty(1, dtype=torch.float64, device=handle.device)   # the C ABI writes device memory, never syncs
    _lib.check(L.b2d_trustworthiness_score(handle.stream_ptr, out.data_ptr(), x_cai.data, m, e_cai.data, d, n, m, d,
                                           int(n_neighbors), mt, int(batch_size), ws.data_ptr(), ws.numel()))
    handle.sync()
    return float(out.item())
