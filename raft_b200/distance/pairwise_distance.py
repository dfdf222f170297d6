"""pairwise_distance -- host-side mirror of ``pylibraft.distance.pairwise_distance``
(removed from the reference snapshot, CHANGELOG.md:59; API per SURVEY.md 8(b); wrapper
conventions per python/pylibraft/pylibraft/random/rmat_rectangular_generator.pyx:24-69).

Dispatches through the C ABI (include/raft_b200.h: b2d_pairwise_distance) into the sm_90a
kernels.  No CPU fallback."""
from __future__ import annotations

import numpy as np

from .. import _lib
from ..common import auto_convert_output, auto_sync_handle, cai_wrapper, device_ndarray
from .distance_type import DistanceType, resolve_metric

_DT = {np.dtype(np.float32): _lib.B2D_F32, np.dtype(np.float16): _lib.B2D_F16, np.dtype(np.float64): _lib.B2D_F64}


def _layout(w: cai_wrapper):
    """(row_major, leading dimension in elements) of a 2-D device array."""
    it = w.dtype.itemsize
    r, c = w.shape
    s0, s1 = w.strides
    if (s1 == it or c == 1) and s0 % it == 0 and s0 >= c * it or r == 1 and s1 == it:
        return True, (s0 // it if r > 1 else max(c, 1))
    if (s0 == it or r == 1) and s1 % it == 0 and s1 >= r * it:
        return False, (s1 // it if c > 1 else max(r, 1))
    raise ValueError("Inputs must be C- or F-contiguous (optionally with a padded leading dimension)")


def pairwise_distance_raw(stream_ptr, metric, x_ptr, ldx, y_ptr, ldy, out_ptr, ldd, m, n, k,
                          row_major, p, ws_ptr, ws_bytes, dtype=_lib.B2D_F32):
    """Thin 1:1 call of the C ABI with raw device pointers (what a cgo/Cython binding does)."""
    L = _lib.lib()
    _lib.check(L.b2d_pairwise_distance(stream_ptr, int(metric), dtype, x_ptr, ldx, y_ptr, ldy, out_ptr,
                                       ldd, m, n, k, 1 if row_major else 0, float(p), ws_ptr, ws_bytes))


@auto_sync_handle
@auto_convert_output
def pairwise_distance(X, Y, out=None, metric="euclidean", p=2.0, handle=None):
    """Compute pairwise distances between X [m,k] and Y [n,k].

    Parameters mirror pylibraft: X, Y any ``__cuda_array_interface__`` objects of the same
    float32 / float64 (or float16) dtype and memory order; ``out`` optional [m,n] array of the inputs' dtype (float32 for
    float16 inputs; written in
    place and returned); ``metric`` a string from ``DISTANCE_TYPES`` or a ``DistanceType``;
    ``p`` the Minkowski exponent; ``handle`` a ``DeviceResources`` (None: one is created and
    synchronised before returning)."""
    x_cai, y_cai, d_cai, dists, row_major, ldx, ldy, ldd = _operands(X, Y, out)
    mt = resolve_metric(metric)
    m, k = x_cai.shape
    n = y_cai.shape[0]

    L = _lib.lib()
    dt = _DT[x_cai.dtype]
    need = L.b2d_pairwise_workspace_bytes(int(mt), dt, m, n, k)
    if need == 2 ** 64 - 1:
        raise ValueError("metric %s is not supported for dtype %s" % (metric, x_cai.dtype))
    ws = handle.workspace(need)
    pairwise_distance_raw(handle.stream_ptr, mt, x_cai.data, ldx, y_cai.data, ldy, d_cai.data, ldd,
                          m, n, k, row_major, p, ws.data_ptr(), ws.numel(), dtype=dt)
    return dists


def _operands(X, Y, out):
    """The checked operands of an [m,n] result of X [m,k] and Y [n,k] (pairwise_distance, gram_matrix):
    (x, y, out wrappers, the out array, row_major, ldx, ldy, ldo).  ``out`` None: a new array in the inputs' order."""
    x_cai, y_cai = cai_wrapper(X), cai_wrapper(Y)
    x_cai.validate_shape_dtype(expected_dims=2)
    y_cai.validate_shape_dtype(expected_dims=2)
    m, k = x_cai.shape
    n, ky = y_cai.shape
    if k != ky:
        raise ValueError("Inputs must have same number of columns. a=%s, b=%s" % (k, ky))
    if x_cai.dtype != y_cai.dtype:
        raise TypeError("Inputs must have the same dtypes")
    if x_cai.dtype not in _DT:
        raise TypeError("dtype %s not supported" % x_cai.dtype)

    x_rm, ldx = _layout(x_cai)
    y_rm, ldy = _layout(y_cai)
    if m > 1 and n > 1 and k > 1 and x_rm != y_rm:
        raise ValueError("Inputs must have matching strides")
    row_major = x_rm if (m > 1 and k > 1) else y_rm if (n > 1 and k > 1) else True
    if not row_major:  # degenerate shapes report both orders; recompute ld for the chosen one
        ldx = x_cai.strides[1] // x_cai.dtype.itemsize if k > 1 else max(m, 1)
        ldy = y_cai.strides[1] // y_cai.dtype.itemsize if k > 1 else max(n, 1)
        ldx, ldy = max(ldx, m), max(ldy, n)
    else:
        ldx, ldy = max(ldx, k), max(ldy, k)

    out_dtype = np.float64 if x_cai.dtype == np.dtype(np.float64) else np.float32
    if out is None:
        if row_major:
            dists = device_ndarray.empty((m, n), dtype=out_dtype)
        else:
            import torch
            dists = device_ndarray(torch.empty((n, m), dtype=torch.float64 if out_dtype == np.float64 else torch.float32,
                                               device="cuda").t())
    else:
        dists = out
    d_cai = cai_wrapper(dists)
    d_cai.validate_shape_dtype(expected_dims=2, expected_dtype=out_dtype)
    if d_cai.shape != (m, n):
        raise ValueError("out must have shape (%d, %d)" % (m, n))
    d_rm, ldd = _layout(d_cai)
    if m > 1 and n > 1 and d_rm != row_major:
        raise ValueError("out must have the same memory order as the inputs")
    if not row_major:  # a single row reports C order with a pitch of n; in Fortran order its pitch is the column stride
        ldd = d_cai.strides[1] // d_cai.dtype.itemsize if n > 1 else max(m, 1)
    ldd = max(ldd, n if row_major else m)
    return x_cai, y_cai, d_cai, dists, row_major, ldx, ldy, ldd


# alias kept by the reference for backwards compatibility
distance = pairwise_distance
