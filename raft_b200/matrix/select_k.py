"""raft::matrix::select_k -- exact per-row top-k (cpp/include/raft/matrix/select_k.cuh:72-106), the selection step of a
brute-force kNN for any metric of pairwise_distance and any k."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper


def _output(out, shape, dtype, name, handle):
    if out is None:
        with torch.cuda.stream(handle.torch_stream):
            t = torch.empty(shape, dtype=dtype, device=handle.device)
        return t, t.data_ptr()
    o = cai_wrapper(out)
    o.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32 if dtype == torch.float32 else np.int64)
    if o.shape != shape:
        raise ValueError("%s must have shape %s, got %s" % (name, shape, o.shape))
    if not o.c_contiguous:
        raise _lib.LogicError("%s must be C contiguous" % name)
    return out, o.data


@auto_sync_handle
def select_k(dataset, k=None, distances=None, indices=None, select_min=True, in_idx=None, handle=None):
    """Returns ``(distances float32 [rows, k], indices int64 [rows, k])``: the k smallest (``select_min``) or largest
    values of every row of the C-contiguous float32 device matrix ``dataset`` and their column positions, or the
    entries of ``in_idx`` (int64 [rows, len]) at those positions.

    Signature of the historical ``pylibraft.matrix.select_k`` [RECALLED] plus ``in_idx``.  ``distances`` / ``indices``:
    optional preallocated C-contiguous outputs, written in place (k is then read from their shape).  Order: -0.0 and
    +0.0 are equal and every NaN ranks above +inf; equal values go to the smaller column.  Every row is sorted, best
    first.  The values are the input bits unchanged.  k outside [1, len] or a non-contiguous input raises LogicError."""
    x = cai_wrapper(dataset)
    x.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if not x.c_contiguous:
        raise _lib.LogicError("dataset must be C contiguous")
    rows, length = x.shape
    if k is None:
        if distances is not None:
            k = cai_wrapper(distances).shape[1]
        elif indices is not None:
            k = cai_wrapper(indices).shape[1]
        else:
            raise ValueError("Argument k must be specified if both distances and indices are None")
    k = int(k)
    idx_ptr = None
    if in_idx is not None:
        ii = cai_wrapper(in_idx)
        ii.validate_shape_dtype(expected_dims=2, expected_dtype=np.int64)
        if ii.shape != (rows, length):
            raise ValueError("in_idx must have the shape of dataset %s, got %s" % ((rows, length), ii.shape))
        if not ii.c_contiguous:
            raise _lib.LogicError("in_idx must be C contiguous")
        idx_ptr = ii.data
    L = _lib.lib()
    need = L.b2d_select_k_workspace_bytes(rows, length, k)
    if need == 2 ** 64 - 1:
        raise _lib.LogicError("k = %d must be in [1, len = %d]" % (k, length))
    dist, dist_ptr = _output(distances, (rows, k), torch.float32, "distances", handle)
    idx, out_idx_ptr = _output(indices, (rows, k), torch.int64, "indices", handle)
    ws = handle.workspace(need)
    _lib.check(L.b2d_select_k(handle.stream_ptr, x.data, length, idx_ptr, rows, length, k, 1 if select_min else 0,
                              dist_ptr, out_idx_ptr, ws.data_ptr(), ws.numel()))
    return dist, idx
