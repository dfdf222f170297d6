"""mean_shift -- sklearn.cluster.MeanShift on the fused epsilon neighbourhood (DBSCAN's rule) with the neighbour sums on
the tensor cores.  Dispatches through the C ABI (include/raft_b200.h: b2d_mean_shift_fit).  A project API: pylibraft
never had this entry point, so there is no pylibraft alias."""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper

MeanShiftOutput = namedtuple("MeanShiftOutput", "cluster_centers labels n_iter")

MAX_D = 320   # the whole distance of a pair is formed at once


def _rows(cai, name):
    """(rows, cols, row pitch in elements) of a float32 matrix whose rows are contiguous"""
    cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    r, c = cai.shape
    if r > 1 and c > 1 and cai.strides[1] != 4:
        raise ValueError("%s must have contiguous rows (row-major, any row pitch)" % name)
    ld = cai.strides[0] // 4 if r > 1 else c
    if (r > 1 and cai.strides[0] % 4) or ld < c:
        raise ValueError("%s has a row pitch below its row length" % name)
    return r, c, max(ld, c)


@auto_sync_handle
def estimate_bandwidth(X, quantile=0.3, handle=None):
    """sklearn.cluster.estimate_bandwidth(X, quantile=quantile) without subsampling: the mean over the rows of X of the
    Euclidean distance to the max(1, floor(n * quantile))-th nearest row, the row itself counted (at distance 0).
    Composed from ``pairwise_distance`` row slabs and ``select_k``; returns a float."""
    from ..distance import pairwise_distance
    from ..matrix import select_k
    x = torch.as_tensor(X, device=handle.device)
    if x.dim() != 2 or x.dtype != torch.float32:
        raise ValueError("X must be a float32 matrix")
    n = x.shape[0]
    if n == 0:
        raise ValueError("X has no rows")
    if not 0.0 <= float(quantile) <= 1.0:
        raise ValueError("quantile must be in [0, 1], got %r" % (quantile,))
    k = max(1, int(n * quantile))
    slab = max(1, min(n, (1 << 28) // max(n, 1)))   # about 1 GiB of distances per slab
    total = 0.0
    with torch.cuda.stream(handle.torch_stream):
        for r0 in range(0, n, slab):
            d = torch.as_tensor(pairwise_distance(x[r0:r0 + slab], x, metric="euclidean", handle=handle),
                                device=handle.device)
            vals, _ = select_k(d, k=k, handle=handle)
            total += float(torch.as_tensor(vals, device=handle.device)[:, k - 1].double().sum().item())
    return total / n


@auto_sync_handle
def mean_shift(X, bandwidth=None, seeds=None, bin_seeding=False, min_bin_freq=1, cluster_all=True, max_iter=300,
               max_mbytes_per_batch=None, handle=None):
    """Mean shift of the rows of X (float32 [n, d] on the device, rows contiguous, any row pitch >= d, d <= 320):
    ``sklearn.cluster.MeanShift(bandwidth, seeds=seeds, bin_seeding=bin_seeding, min_bin_freq=min_bin_freq,
    cluster_all=cluster_all, max_iter=max_iter).fit(X)`` with the neighbourhood test ``dist <= bandwidth`` decided by the
    engine's squared distance against fp32(bandwidth^2), as ``dbscan`` decides it.

    bandwidth None is ``estimate_bandwidth(X)``.  seeds: float32 [s, d] on the device (bin_seeding is then ignored).
    ``max_mbytes_per_batch`` (MiB, default 1024) bounds the adjacency formed at once; the result does not depend on it,
    nor on the order of the seeds.

    Returns ``MeanShiftOutput(cluster_centers, labels, n_iter)``: float32 [n_centers, d] and int32 [n] torch tensors on
    the device (-1: a row farther than bandwidth from every centre, with cluster_all=False) and the largest iteration
    count of any seed.  Raises ValueError when no seed has a neighbour, as sklearn does."""
    x = cai_wrapper(X)
    n, d, ldx = _rows(x, "X")
    if n == 0:
        raise ValueError("X has no rows")
    if d > MAX_D:
        raise _lib.LogicError("mean_shift supports d <= %d, got %d" % (MAX_D, d))
    if bandwidth is None:
        bandwidth = estimate_bandwidth(X, handle=handle)
    bandwidth = float(bandwidth)
    if not bandwidth > 0.0:
        raise ValueError("bandwidth needs to be greater than zero or None, got %f" % bandwidth)
    sp, ns, lds = None, 0, d
    if seeds is not None:
        sc = cai_wrapper(seeds)
        ns, sd, lds = _rows(sc, "seeds")
        if sd != d:
            raise ValueError("seeds must have %d columns, got %d" % (d, sd))
        if ns == 0:
            raise ValueError("seeds has no rows")
        sp = sc.data
    if int(max_iter) < 0:
        raise _lib.LogicError("max_iter must be >= 0, got %r" % (max_iter,))
    if bin_seeding and seeds is None and int(min_bin_freq) < 1:
        raise _lib.LogicError("min_bin_freq must be >= 1, got %r" % (min_bin_freq,))
    mb = 0 if max_mbytes_per_batch is None else int(max_mbytes_per_batch * (1 << 20))
    cap = ns if seeds is not None else n
    with torch.cuda.stream(handle.torch_stream):
        centers = torch.empty((cap, d), dtype=torch.float32, device=handle.device)
        labels = torch.empty((n,), dtype=torch.int32, device=handle.device)
        out = torch.zeros((2,), dtype=torch.int32, device=handle.device)   # n_centers, n_iter
    L = _lib.lib()
    need = L.b2d_mean_shift_fit_workspace_bytes(n, d, ns, mb)
    ws = handle.workspace(need if need != 2 ** 64 - 1 else 0)
    _lib.check(L.b2d_mean_shift_fit(handle.stream_ptr, x.data, ldx, n, d, bandwidth, sp, lds, ns,
                                    1 if bin_seeding else 0, int(min_bin_freq), 1 if cluster_all else 0, int(max_iter), mb,
                                    centers.data_ptr(), out.data_ptr(), labels.data_ptr(), out.data_ptr() + 4,
                                    ws.data_ptr(), ws.numel()))
    handle.sync()
    n_centers, n_iter = (int(v) for v in out.cpu().tolist())
    if n_centers == 0:
        raise ValueError("No point was within bandwidth=%f of any seed. Try a different seeding strategy or increase "
                         "the bandwidth." % bandwidth)
    return MeanShiftOutput(centers[:n_centers], labels, n_iter)
