"""kernel_density -- the log density of each query row under a kernel density estimate of the dataset rows (the answer of
``sklearn.neighbors.KernelDensity(atol=0, rtol=0).fit(dataset, sample_weight=...).score_samples(queries)``), fused into
the tensor-core distance kernel so the m x n distance matrix is never written (raft_b200/csrc/kde.cu, expanded_tc.cuh
EPI_KDE).  A project API: pylibraft never had this entry point, so there is no pylibraft alias."""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper

KERNELS = ("gaussian", "tophat", "epanechnikov", "exponential", "linear", "cosine")   # B2D_KDE_* order
MAX_D = 320   # the whole distance of a pair is formed at once


def bandwidth_of(bandwidth, n, d):
    """The bandwidth sklearn's KernelDensity.fit uses for n dataset rows of d columns: a number as given, or the rule
    "scott" (n^(-1 / (d + 4))) or "silverman" ((n (d + 2) / 4)^(-1 / (d + 4)))."""
    if isinstance(bandwidth, str):
        if bandwidth == "scott":
            return n ** (-1 / (d + 4))
        if bandwidth == "silverman":
            return (n * (d + 2) / 4) ** (-1 / (d + 4))
        raise ValueError("bandwidth must be a number, 'scott' or 'silverman', got %r" % bandwidth)
    return float(bandwidth)


def _rows(cai, name):
    """(rows, cols, row pitch in elements) of a float32 matrix whose rows are contiguous"""
    cai.validate_shape_dtype(expected_dims=2, expected_dtype=np.float32)
    r, c = cai.shape
    if c > 1 and cai.strides[1] != 4:
        raise ValueError("%s must have contiguous rows (row-major, any row pitch)" % name)
    ld = cai.strides[0] // 4 if r > 1 else c
    if cai.strides[0] % 4 or ld < c:
        raise ValueError("%s has a row pitch below its row length" % name)
    return r, c, max(ld, c)


@auto_sync_handle
def kernel_density(dataset, queries, bandwidth=1.0, kernel="gaussian", sample_weight=None, batch_cols=0, handle=None):
    """Returns the float64 torch tensor [m] of ``log(sum_j w_j K(|q_i - x_j|; h) / sum_j w_j) + log_norm(kernel, h, d)``.

    dataset [n, d] and queries [m, d]: float32 ``__cuda_array_interface__`` objects with contiguous rows (a row pitch is
    allowed), d <= 320.  kernel: one of "gaussian", "tophat", "epanechnikov", "exponential", "linear", "cosine" (sklearn's
    kernels); the compact ones count the pairs with d^2 < fp32(h^2) only.  bandwidth: h > 0, or "scott" / "silverman"
    (sklearn's rules in n and d).  sample_weight: optional float32 [n] on the device, finite and >= 0 with a positive
    total; a weight of 0 removes its row.  A bad weight raises ValueError; checking costs one host read.

    d^2 is bit for bit the float32 value ``pairwise_distance(queries, dataset, "sqeuclidean")`` returns, including its rule
    that a row paired with itself is at 0 when ``queries`` is ``dataset`` (a copy gets no such rule).  The result equals
    sklearn's score_samples with atol = rtol = 0, except for the cosine kernel at even d, where sklearn's normalisation
    is wrong and this one is exact.  Gaussian and exponential are evaluated as a log-sum-exp, so a query far from the data
    keeps a finite log density; a compact kernel with no dataset row in its support gives -inf.  A NaN distance makes
    its query's result NaN.  The result is the same bits on every call and for every ``batch_cols`` (dataset columns per
    pass, rounded up to 256; 0 keeps the per-pass scratch at about 1 GiB)."""
    if kernel not in KERNELS:
        raise ValueError("kernel must be one of %s, got %r" % (", ".join(KERNELS), kernel))
    d_cai, q_cai = cai_wrapper(dataset), cai_wrapper(queries)
    n, dim, ldy = _rows(d_cai, "dataset")
    m, dq, ldx = _rows(q_cai, "queries")
    if dim != dq:
        raise ValueError("Inputs must have same number of columns. a=%s, b=%s" % (dim, dq))
    if dim > MAX_D:
        raise _lib.LogicError("kernel_density supports d <= %d, got d = %d" % (MAX_D, dim))
    h = bandwidth_of(bandwidth, n, dim)
    w_ptr = None
    if sample_weight is not None:
        w_cai = cai_wrapper(sample_weight)
        w_cai.validate_shape_dtype(expected_dims=1, expected_dtype=np.float32)
        if w_cai.shape[0] != n or not w_cai.c_contiguous:
            raise ValueError("sample_weight must be a contiguous float32 vector of %d entries" % n)
        with torch.cuda.stream(handle.torch_stream):
            w = torch.as_tensor(sample_weight, device=handle.device)
            bad = bool((~torch.isfinite(w) | (w < 0)).any() | ~(w > 0).any())   # the one host read
        if bad:
            raise ValueError("sample_weight must be finite and >= 0, with a positive total")
        w_ptr = w_cai.data
    L = _lib.lib()
    with torch.cuda.stream(handle.torch_stream):
        out = torch.empty(m, dtype=torch.float64, device=handle.device)
    ws = handle.workspace(L.b2d_kde_workspace_bytes(m, n, dim, int(batch_cols)))
    _lib.check(L.b2d_kde_score_samples(handle.stream_ptr, KERNELS.index(kernel), h, d_cai.data, ldy, w_ptr, q_cai.data,
                                       ldx, m, n, dim, int(batch_cols), out.data_ptr(), ws.data_ptr(), ws.numel()))
    return out
