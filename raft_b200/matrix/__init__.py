"""raft::matrix::argmin -- the separate-pass row arg-min (cpp/include/raft/matrix/argmin.cuh:25-37), SURVEY.md 8(a9) --
and raft::matrix::select_k, the exact per-row top-k (select_k.py)."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from .select_k import select_k  # noqa: F401


@auto_sync_handle
def argmin(X, out=None, handle=None):
    """Column index (int32 [rows]) of the minimum of every row of the C-contiguous float32 device matrix X;
    ties go to the smaller index (cub::ArgMin, cpp/include/raft/matrix/detail/math.cuh:290-343)."""
    x = cai_wrapper(X)
    x.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    if not x.c_contiguous:
        raise ValueError("Input must be C contiguous")
    rows, n = x.shape
    with torch.cuda.stream(handle.torch_stream):
        if out is None:
            out = torch.empty(rows, dtype=torch.int32, device=handle.device)
    o = cai_wrapper(out)
    o.validate_shape_dtype(expected_dims=1, expected_dtype=np.int32)
    if o.shape[0] != rows:
        raise ValueError("out must have shape (%d,)" % rows)
    _lib.check(_lib.lib().b2d_row_argmin(handle.stream_ptr, o.data, x.data, n, rows, n))
    return out
