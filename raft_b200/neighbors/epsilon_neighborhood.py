"""raft::neighbors::epsilon_neighborhood::eps_neighbors_l2sq -- the epsilon neighbourhood of the rows of X among the rows of
Y under the squared L2 distance (the vertex-degree step of DBSCAN), fused into the tensor-core distance kernel so the
m x n distance matrix is never written."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper

MAX_K = 320   # the whole distance of a pair is formed at once


@auto_sync_handle
def eps_neighbors_l2sq(x, y, eps, adj=None, vd=None, return_adj=True, handle=None):
    """Returns ``(adj, vd)``: ``adj`` bool [m, n] with ``adj[i, j] = ||x_i - y_j||^2 <= eps`` (None when ``return_adj`` is
    False: count only), and ``vd`` [n + 1] with ``vd[j]`` = the number of rows i adjacent to column j and ``vd[n]`` the
    total (per-column degrees, as the reference's kernel computed them).

    x [m, k], y [n, k]: C-contiguous float32 device arrays, k <= 320 (LogicError otherwise).  eps is the SQUARED radius.
    The distance is exactly the one ``pairwise_distance(x, y, "sqeuclidean")`` returns, so ``adj`` equals that matrix
    compared with eps.  When y is x, or a view of a window of its rows, a row's pair with itself is adjacent for every
    eps >= 0; a copy of x elsewhere in memory gets no such rule.  A NaN distance is never adjacent.
    adj: optional preallocated bool / uint8 [m, n] output with contiguous rows (any row pitch >= n).  vd: optional
    preallocated int64 or int32 [n + 1] output (an int32 count wraps modulo 2^32).  The counts are always zeroed first."""
    xc, yc = cai_wrapper(x), cai_wrapper(y)
    xc.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    yc.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if xc.shape[1] != yc.shape[1]:
        raise ValueError("Inputs must have same number of columns. a=%s, b=%s" % (xc.shape[1], yc.shape[1]))
    if not (xc.c_contiguous and yc.c_contiguous):
        raise ValueError("Inputs must be C contiguous")
    m, k = xc.shape
    n = yc.shape[0]
    if k > MAX_K:
        raise _lib.LogicError("eps_neighbors_l2sq supports k <= %d, got k = %d" % (MAX_K, k))
    with torch.cuda.stream(handle.torch_stream):
        if vd is None:
            vd = torch.empty(n + 1, dtype=torch.int64, device=handle.device)
        vd_t = torch.as_tensor(vd, device=handle.device)
        if vd_t.dtype not in (torch.int32, torch.int64) or vd_t.shape != (n + 1,) or not vd_t.is_contiguous():
            raise ValueError("vd must be a contiguous int32 or int64 array of shape (%d,)" % (n + 1))
        adj_ptr, ld_adj = None, n
        if return_adj:
            if adj is None:
                adj = torch.empty((m, n), dtype=torch.bool, device=handle.device)
            a = torch.as_tensor(adj, device=handle.device)
            if a.dtype not in (torch.bool, torch.uint8) or a.shape != (m, n):
                raise ValueError("adj must be bool or uint8 of shape (%d, %d)" % (m, n))
            if n > 1 and a.stride(1) != 1:
                raise ValueError("adj must be row-major with contiguous rows")
            ld_adj = a.stride(0) if m > 1 else n
            adj_ptr = a.data_ptr()
        else:
            adj = None
    L = _lib.lib()
    ws = handle.workspace(L.b2d_eps_neighbors_l2sq_workspace_bytes(m, n, k))
    _lib.check(L.b2d_eps_neighbors_l2sq(handle.stream_ptr, adj_ptr, ld_adj, vd_t.data_ptr(),
                                        1 if vd_t.dtype == torch.int64 else 0, 1, xc.data, k, yc.data, k, m, n, k,
                                        float(eps), ws.data_ptr(), ws.numel()))
    return adj, vd
