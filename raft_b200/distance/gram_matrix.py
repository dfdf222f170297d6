"""gram_matrix -- the kernel Gram matrices of the removed ``raft::distance::kernels`` (GramMatrixBase, PolynomialKernel,
RBFKernel, TanhKernel), the kernel evaluations of cuML's SVM.  Dispatches through the C ABI (include/raft_b200.h:
b2d_gram_matrix): the transform runs in the epilogue of the distance kernel, so the m x n matrix is written once."""
from __future__ import annotations

import math

from .. import _lib
from ..common import auto_convert_output, auto_sync_handle
from .pairwise_distance import _DT, _operands

KERNEL_TYPES = {
    "linear": _lib.B2D_KERNEL_LINEAR,
    "polynomial": _lib.B2D_KERNEL_POLYNOMIAL,
    "rbf": _lib.B2D_KERNEL_RBF,
    "tanh": _lib.B2D_KERNEL_TANH,
}


@auto_sync_handle
@auto_convert_output
def gram_matrix(X, Y, kernel="rbf", degree=3, gamma=1.0, coef0=0.0, out=None, handle=None):
    """Kernel matrix of X [m,k] and Y [n,k]:

    - ``"linear"``:     <x_i, y_j> (the same values as ``pairwise_distance(X, Y, "inner_product")``)
    - ``"polynomial"``: (gamma <x_i, y_j> + coef0) ** degree, integer degree >= 0 (degree 0: 1 everywhere)
    - ``"rbf"``:        exp(-gamma ||x_i - y_j||^2); when Y is X the diagonal is exactly 1
    - ``"tanh"``:       tanh(gamma <x_i, y_j> + coef0)

    X, Y: any ``__cuda_array_interface__`` objects of one float32 / float16 / float64 dtype and one memory order (C or
    Fortran, optionally with a padded leading dimension).  ``out``: optional [m,n] array in that order, float64 for
    float64 inputs and float32 otherwise (written in place and returned); by default a new ``device_ndarray``.  gamma and
    coef0 are used in float32 for float32 / float16 inputs and in float64 for float64 inputs; degree is read for
    ``"polynomial"`` only.  ``handle``: a ``DeviceResources`` (None: one is created and synchronised before returning)."""
    if kernel not in KERNEL_TYPES:
        raise ValueError("kernel must be one of %s, got %r" % (sorted(KERNEL_TYPES), kernel))
    kt = KERNEL_TYPES[kernel]
    if kt == _lib.B2D_KERNEL_POLYNOMIAL:
        if int(degree) != degree or degree < 0:
            raise ValueError("degree must be an integer >= 0, got %r" % (degree,))
    if not (math.isfinite(gamma) and math.isfinite(coef0)):
        raise ValueError("gamma and coef0 must be finite")
    x_cai, y_cai, o_cai, res, row_major, ldx, ldy, ldo = _operands(X, Y, out)
    m, k = x_cai.shape
    n = y_cai.shape[0]
    L = _lib.lib()
    dt = _DT[x_cai.dtype]
    ws = handle.workspace(L.b2d_gram_matrix_workspace_bytes(kt, dt, m, n, k))
    _lib.check(L.b2d_gram_matrix(handle.stream_ptr, kt, int(degree) if kt == _lib.B2D_KERNEL_POLYNOMIAL else 0,
                                 float(gamma), float(coef0), dt, x_cai.data, ldx, y_cai.data, ldy, o_cai.data, ldo, m, n, k,
                                 1 if row_major else 0, ws.data_ptr(), ws.numel()))
    return res
