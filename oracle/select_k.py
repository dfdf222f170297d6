"""TEST INFRASTRUCTURE ONLY -- numpy restatement of raft::matrix::select_k as this project defines it (DESIGN.md K9).

Order: the IEEE float order with -0.0 == +0.0 and every NaN (either sign bit) above +inf; select_min takes the
smallest, otherwise the largest (so NaNs come first, cpp/tests/matrix/select_k_edgecases.cu).  Equal values go to the
smaller column in both directions.  Each row of the result is sorted best first, equal values by ascending column, and
the returned values are the input bits unchanged.

Written independently of the CUDA key (raft_b200/csrc/select_k.cuh): the special values are found with numpy's float
predicates (isnan, < 0, == 0), not bit tests, and the selection is numpy's partition and sort."""
from __future__ import annotations

import numpy as np


def select_key(values, select_min=True):
    """uint32 key of every element: ascending key order is the selection order (ties: equal keys)."""
    v = np.ascontiguousarray(values, dtype=np.float32)
    b = v.view(np.uint32)
    nan = np.isnan(v)
    key = np.where(v < 0, ~b, b | np.uint32(0x80000000)).astype(np.uint32)   # ordered bits of the non-NaN values
    key[v == 0] = np.uint32(0x80000000)                                       # -0.0 == +0.0
    key[nan] = np.uint32(0xFFFFFFFF)                                          # every NaN above +inf
    return key if select_min else ~key


def select_k(values, k, select_min=True, in_idx=None):
    """(values float32 [rows, k], indices int64 [rows, k]) of the k best elements of every row of values [rows, len];
    indices are columns, or in_idx[row, column] when in_idx is given."""
    v = np.ascontiguousarray(values, dtype=np.float32)
    if v.ndim != 2:
        raise ValueError("values must be 2-d")
    rows, n = v.shape
    k = int(k)
    if not 1 <= k <= n:
        raise ValueError("k must be in [1, len]")
    # (key, column) as one unique 64-bit word: its order is the selection order with the column tie rule
    words = (select_key(v, select_min).astype(np.uint64) << np.uint64(32)) | np.arange(n, dtype=np.uint64)[None, :]
    if k < n:
        words = np.partition(words, k - 1, axis=1)[:, :k]
    words = np.sort(words, axis=1)
    cols = (words & np.uint64(0xFFFFFFFF)).astype(np.int64)
    out_v = np.take_along_axis(v, cols, axis=1)
    out_i = cols if in_idx is None else np.take_along_axis(np.asarray(in_idx, dtype=np.int64), cols, axis=1)
    return out_v, out_i
