"""CPU fp64 restatement of raft::distance::pairwise_distance / fusedL2NN (TEST INFRASTRUCTURE).

Header: see oracle/__init__.py ("parity unpinned").  Every function cites the reference
file:line it follows; where the reference source was deleted upstream the citation is the
surviving evidence listed in SURVEY.md section 8(a).
"""
from __future__ import annotations

import enum
import numpy as np

__all__ = [
    "DistanceType", "pairwise_distance", "fused_l2_nn", "row_norm_sq", "argmin_op",
    "row_argmin", "compare_approx", "match_approx", "make_blobs", "EXPANDED", "UNEXPANDED",
    "pack_minloc", "unpack_minloc", "knn_l2", "knn", "silhouette_score", "trustworthiness_score",
]


class DistanceType(enum.IntEnum):
    """raft::distance::DistanceType (enum values: SURVEY.md 8(a1); type name proven by
    cpp/include/raft/stats/silhouette_score.cuh:45)."""
    L2Expanded = 0
    L2SqrtExpanded = 1
    CosineExpanded = 2
    L1 = 3
    L2Unexpanded = 4
    L2SqrtUnexpanded = 5
    InnerProduct = 6
    Linf = 7
    Canberra = 8
    LpUnexpanded = 9
    CorrelationExpanded = 10
    JaccardExpanded = 11
    HellingerExpanded = 12
    Haversine = 13
    BrayCurtis = 14
    JensenShannon = 15
    HammingUnexpanded = 16
    KLDivergence = 17
    RusselRaoExpanded = 18
    DiceExpanded = 19
    Precomputed = 100


EXPANDED = (DistanceType.L2Expanded, DistanceType.L2SqrtExpanded, DistanceType.CosineExpanded,
            DistanceType.CorrelationExpanded, DistanceType.InnerProduct, DistanceType.HellingerExpanded,
            DistanceType.RusselRaoExpanded, DistanceType.JaccardExpanded, DistanceType.DiceExpanded)
UNEXPANDED = (DistanceType.L1, DistanceType.L2Unexpanded, DistanceType.L2SqrtUnexpanded,
              DistanceType.Linf, DistanceType.Canberra, DistanceType.LpUnexpanded,
              DistanceType.HammingUnexpanded, DistanceType.KLDivergence, DistanceType.JensenShannon,
              DistanceType.BrayCurtis)


def row_norm_sq(x: np.ndarray) -> np.ndarray:
    """Squared L2 row norm, fp64 (spec: cpp/include/raft/linalg/norm.cuh:50-58, L2Norm =
    sum of squares, naive check cpp/tests/linalg/norm.cu:42-66)."""
    x = np.asarray(x, dtype=np.float64)
    return np.einsum("ij,ij->i", x, x)


def _block(x64, y64, metric, p):
    if metric in (DistanceType.L2Expanded, DistanceType.L2SqrtExpanded,
                  DistanceType.L2Unexpanded, DistanceType.L2SqrtUnexpanded):
        # mathematically identical; fp64 expanded form is exact enough to be the oracle,
        # but use the difference form for robustness to cancellation.
        xn = np.einsum("ij,ij->i", x64, x64)
        yn = np.einsum("ij,ij->i", y64, y64)
        d = xn[:, None] + yn[None, :] - 2.0 * (x64 @ y64.T)
        # fp64 cancellation error is ~1e-16*|x|^2, far below the 1e-4 bar; clamp like the
        # reference epilogue does (SURVEY.md 8(a3): "clamp <0 -> 0").
        np.maximum(d, 0.0, out=d)
        if metric in (DistanceType.L2SqrtExpanded, DistanceType.L2SqrtUnexpanded):
            np.sqrt(d, out=d)
        return d
    if metric == DistanceType.InnerProduct:
        return x64 @ y64.T
    if metric == DistanceType.CosineExpanded:
        xn = np.sqrt(np.einsum("ij,ij->i", x64, x64))
        yn = np.sqrt(np.einsum("ij,ij->i", y64, y64))
        with np.errstate(divide="ignore", invalid="ignore"):
            return 1.0 - (x64 @ y64.T) / (xn[:, None] * yn[None, :])
    if metric == DistanceType.CorrelationExpanded:
        # 1 - (k*sum(xy) - sum(x)sum(y)) / sqrt((k*sum(x^2)-sum(x)^2)(k*sum(y^2)-sum(y)^2))
        # (SURVEY.md 8(a3)); computed on centred rows, which is the same quantity.
        xc = x64 - x64.mean(axis=1, keepdims=True)
        yc = y64 - y64.mean(axis=1, keepdims=True)
        xn = np.sqrt(np.einsum("ij,ij->i", xc, xc))
        yn = np.sqrt(np.einsum("ij,ij->i", yc, yc))
        with np.errstate(divide="ignore", invalid="ignore"):
            return 1.0 - (xc @ yc.T) / (xn[:, None] * yn[None, :])
    # SURVEY.md 8(f) item 4 metrics.  [RECALLED] definitions of the removed reference ops:
    #   Hellinger  sqrt(max(0, 1 - sum sqrt(x_i) sqrt(y_i)))        RusselRao  (k - sum x_i y_i) / k
    #   Hamming    (# x_i != y_i) / k                               JensenShannon  sqrt(0.5 sum x log(x/m) + y log(y/m))
    #   KLDivergence  0.5 * sum x_i log(x_i / y_i)  (the 0.5 is the reference's epilogue, not scipy's)
    if metric == DistanceType.HellingerExpanded:
        return np.sqrt(np.maximum(1.0 - np.sqrt(x64) @ np.sqrt(y64).T, 0.0))
    if metric == DistanceType.RusselRaoExpanded:
        k = x64.shape[1]
        return (k - x64 @ y64.T) / k
    if metric in (DistanceType.JaccardExpanded, DistanceType.DiceExpanded):
        # [RECALLED] expanded forms on a = <x,y>, s = |x|^2 + |y|^2 (the reference's sparse / dense ops; on
        # indicator data they are scipy's jaccard / dice):  Jaccard 1 - a / (s - a),  Dice 1 - 2a / s;  0/0 -> 0
        a = x64 @ y64.T
        s_ = np.einsum("ij,ij->i", x64, x64)[:, None] + np.einsum("ij,ij->i", y64, y64)[None, :]
        den = s_ - a if metric == DistanceType.JaccardExpanded else s_
        num = a if metric == DistanceType.JaccardExpanded else 2.0 * a
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(den > 0.0, np.maximum(1.0 - num / den, 0.0), 0.0)
    if metric == DistanceType.BrayCurtis:
        with np.errstate(divide="ignore", invalid="ignore"):
            return (np.abs(x64[:, None, :] - y64[None, :, :]).sum(axis=2) /
                    np.abs(x64[:, None, :] + y64[None, :, :]).sum(axis=2))
    if metric == DistanceType.HammingUnexpanded:
        return (x64[:, None, :] != y64[None, :, :]).mean(axis=2)
    if metric in (DistanceType.KLDivergence, DistanceType.JensenShannon):
        a, b = x64[:, None, :], y64[None, :, :]
        with np.errstate(divide="ignore", invalid="ignore"):
            if metric == DistanceType.KLDivergence:
                t = np.where(a == 0.0, 0.0, a * (np.log(a) - np.log(b)))
                return 0.5 * t.sum(axis=2)
            mm = 0.5 * (a + b)
            ta = np.where(a == 0.0, 0.0, a * (np.log(a) - np.log(mm)))
            tb = np.where(b == 0.0, 0.0, b * (np.log(b) - np.log(mm)))
            return np.sqrt(np.maximum(0.5 * (ta + tb).sum(axis=2), 0.0))
    # unexpanded metrics: SURVEY.md 8(a4)
    diff = x64[:, None, :] - y64[None, :, :]
    if metric == DistanceType.L1:
        return np.abs(diff).sum(axis=2)
    if metric == DistanceType.Linf:
        return np.abs(diff).max(axis=2) if diff.shape[2] else np.zeros(diff.shape[:2])
    if metric == DistanceType.Canberra:
        den = np.abs(x64)[:, None, :] + np.abs(y64)[None, :, :]
        with np.errstate(divide="ignore", invalid="ignore"):
            t = np.where(den == 0.0, 0.0, np.abs(diff) / den)   # 0/0 -> 0
        return t.sum(axis=2)
    if metric == DistanceType.LpUnexpanded:
        return (np.abs(diff) ** p).sum(axis=2) ** (1.0 / p)
    raise ValueError(f"metric {metric!r} not on the hot path")


def pairwise_distance(x, y, metric=DistanceType.L2Expanded, metric_arg: float = 2.0,
                      block: int = 256) -> np.ndarray:
    """dist[i,j] = metric(x_i, y_j); x:[m,k], y:[n,k] row-major -> [m,n] fp64.

    Follows raft::distance::pairwise_distance (call shape:
    cpp/include/raft/stats/detail/silhouette_score.cuh:205-206; semantics SURVEY.md 8(a2-a4)).
    Inputs are taken at their own precision (fp32/fp16) and promoted to fp64."""
    metric = DistanceType(metric)
    x64 = np.ascontiguousarray(x, dtype=np.float64)
    y64 = np.ascontiguousarray(y, dtype=np.float64)
    assert x64.ndim == 2 and y64.ndim == 2 and x64.shape[1] == y64.shape[1]
    m, n = x64.shape[0], y64.shape[0]
    out = np.empty((m, n), dtype=np.float64)
    if metric in EXPANDED + (DistanceType.L2Unexpanded, DistanceType.L2SqrtUnexpanded):
        block = max(block, 2048)
    elif metric in (DistanceType.KLDivergence, DistanceType.JensenShannon, DistanceType.HammingUnexpanded,
                    DistanceType.BrayCurtis):
        block = min(block, 128)
    for i0 in range(0, m, block):
        for j0 in range(0, n, block):
            out[i0:i0 + block, j0:j0 + block] = _block(
                x64[i0:i0 + block], y64[j0:j0 + block], metric, float(metric_arg))
    return out


def argmin_op(a, b):
    """raft::argmin_op on (key, value) pairs: cpp/include/raft/core/operators.hpp:187-194."""
    if (b[1] < a[1]) or ((a[1] == b[1]) and (b[0] < a[0])):
        return b
    return a


def row_argmin(mat: np.ndarray) -> np.ndarray:
    """raft::matrix::argmin: cpp/include/raft/matrix/argmin.cuh:25-37 (ties -> smaller
    index, same as np.argmin's first-occurrence rule)."""
    return np.argmin(np.asarray(mat), axis=1).astype(np.int32)


def fused_l2_nn(x, y, sqrt: bool = False, block: int = 4096):
    """out[i] = (argmin_j, min_j) ||x_i - y_j||^2 (or its sqrt), ties -> smaller j.

    Follows raft::distance::fusedL2NN[MinReduce] (SURVEY.md 8(a5); tie-break law
    cpp/include/raft/core/operators.hpp:187-194).  Returns (idx int32[m], val fp64[m])."""
    x64 = np.ascontiguousarray(x, dtype=np.float64)
    y64 = np.ascontiguousarray(y, dtype=np.float64)
    m, n = x64.shape[0], y64.shape[0]
    best_v = np.full(m, np.inf)
    best_i = np.zeros(m, dtype=np.int64)
    for j0 in range(0, n, block):
        d = _block(x64, y64[j0:j0 + block], DistanceType.L2Expanded, 2.0)
        loc = np.argmin(d, axis=1)
        v = d[np.arange(m), loc]
        upd = v < best_v                     # strict: earlier (smaller) index wins ties
        best_v = np.where(upd, v, best_v)
        best_i = np.where(upd, loc + j0, best_i)
    if sqrt:
        best_v = np.sqrt(best_v)
    return best_i.astype(np.int32), best_v


def knn(x, y, n_neighbors: int, metric, block: int = 4096):
    """k nearest rows of y under any metric of pairwise_distance, ascending by (distance, index) -- the
    composition pairwise_distance + select_k(select_min, sorted) (see knn_l2).  Blocked over the columns of y: memory
    O(m * (n_neighbors + block)).  NaN distances sort after every number (then by index), as in one sort of the row."""
    x64 = np.ascontiguousarray(x, dtype=np.float64)
    y64 = np.ascontiguousarray(y, dtype=np.float64)
    m, n = x64.shape[0], y64.shape[0]
    kk = int(n_neighbors)
    best_v = np.empty((m, 0))
    best_i = np.empty((m, 0), dtype=np.int64)
    for j0 in range(0, n, block):
        d = pairwise_distance(x64, y64[j0:j0 + block], metric)
        v = np.concatenate([best_v, d], axis=1)
        i = np.concatenate([best_i, np.broadcast_to(np.arange(j0, j0 + d.shape[1], dtype=np.int64), d.shape)], axis=1)
        order = np.lexsort((i, v), axis=1)[:, :kk]       # primary key: distance, then index
        best_v = np.take_along_axis(v, order, axis=1)
        best_i = np.take_along_axis(i, order, axis=1)
    return best_i, best_v


def knn_l2(x, y, n_neighbors: int, sqrt: bool = False, block: int = 4096):
    """out[i, :] = the n_neighbors rows of y nearest to x_i, ascending by (squared L2 distance, index).

    Restates what the reference's callers composed from raft::distance::pairwise_distance (L2Expanded)
    followed by raft::matrix::select_k(select_min = true, sorted = true)
    (cpp/include/raft/matrix/select_k.cuh:73-106; removed fused form: brute_force::fused_l2_knn,
    CHANGELOG.md:59-60) -- SURVEY.md 8(f2).  Returns (idx int64[m, kk], val fp64[m, kk])."""
    x64 = np.ascontiguousarray(x, dtype=np.float64)
    y64 = np.ascontiguousarray(y, dtype=np.float64)
    m, n = x64.shape[0], y64.shape[0]
    kk = int(n_neighbors)
    best_v = np.full((m, kk), np.inf)
    best_i = np.full((m, kk), np.iinfo(np.int64).max, dtype=np.int64)
    for j0 in range(0, n, block):
        d = _block(x64, y64[j0:j0 + block], DistanceType.L2Expanded, 2.0)
        idx = np.broadcast_to(np.arange(j0, j0 + d.shape[1], dtype=np.int64), d.shape)
        v = np.concatenate([best_v, d], axis=1)
        i = np.concatenate([best_i, idx], axis=1)
        order = np.lexsort((i, v), axis=1)[:, :kk]       # primary key: distance, then index
        best_v = np.take_along_axis(v, order, axis=1)
        best_i = np.take_along_axis(i, order, axis=1)
    if sqrt:
        best_v = np.sqrt(best_v)
    return best_i, best_v


def silhouette_score(x, labels, n_labels=None, metric=None, metric_arg=2.0, return_samples=False):
    """Mean silhouette coefficient, restating raft::stats::silhouette_score
    (cpp/include/raft/stats/detail/silhouette_score.cuh:186-328; per-sample rule SilOp :155-167,
    singleton rule populateAKernel :72-84): a = mean distance to the OTHER members of the own cluster,
    b = min over the other non-empty clusters of the mean distance to it, s = 0 for singleton clusters
    or a == b, else (b - a) / max(a, b).  Default metric = the reference's (L2Unexpanded, squared)."""
    metric = DistanceType.L2Unexpanded if metric is None else metric
    labels = np.asarray(labels)
    n = len(labels)
    n_labels = int(labels.max()) + 1 if n_labels is None else int(n_labels)
    d = pairwise_distance(x, x, metric, metric_arg)
    counts = np.bincount(labels, minlength=n_labels).astype(np.float64)
    sums = np.zeros((n, n_labels))
    for c in range(n_labels):
        sums[:, c] = d[:, labels == c].sum(axis=1)
    own = labels
    a = np.where(counts[own] > 1, sums[np.arange(n), own] / np.maximum(counts[own] - 1, 1), -1.0)
    mean = np.where(counts[None, :] > 0, sums / np.maximum(counts[None, :], 1), np.inf)
    mean[np.arange(n), own] = np.inf
    b = mean.min(axis=1)
    s = np.where((a == -1.0) | (a == b), 0.0, np.where(a > b, (b - a) / np.where(a == 0, 1, a), (b - a) / np.where(b == 0, 1, b)))
    return (float(s.mean()), s) if return_samples else float(s.mean())


def trustworthiness_score(x, x_embedded, n_neighbors: int = 5, metric=None):
    """Restates raft::stats::trustworthiness_score (cpp/include/raft/stats/detail/
    trustworthiness_score.cuh:113-211): the n_neighbors nearest samples j of i in the embedded space (in the caller's
    metric; i itself excluded, ties by index), r(i, j) = position of j in the order of the samples by original-space
    distance from i (i first; ties by index), penalty max(0, r - n_neighbors).  Every sample contributes exactly
    n_neighbors neighbours, also when n_neighbors or more other samples coincide with it in the embedding.  Same value
    as sklearn.manifold.trustworthiness wherever the embedded neighbour set has no ties at its boundary."""
    metric = DistanceType.L2SqrtUnexpanded if metric is None else metric
    x = np.asarray(x, dtype=np.float64)
    e = np.asarray(x_embedded, dtype=np.float64)
    n, k = x.shape[0], int(n_neighbors)
    idx = np.broadcast_to(np.arange(n), (n, n))
    d = pairwise_distance(x, x, metric, 2.0)
    np.fill_diagonal(d, -np.inf)                                   # the sample itself comes first
    order = np.lexsort((idx, d), axis=1)
    rank = np.empty_like(order)
    np.put_along_axis(rank, order, idx, axis=1)
    # run_knn<distance_type> (trustworthiness_score.cuh:79-104): the SAME metric in the embedded space; every L2 form
    # orders like the squared distance, which no square root can merge
    l2 = (DistanceType.L2SqrtUnexpanded, DistanceType.L2Unexpanded, DistanceType.L2Expanded, DistanceType.L2SqrtExpanded)
    de = pairwise_distance(e, e, DistanceType.L2Expanded if metric in l2 else metric, 2.0)
    np.fill_diagonal(de, np.inf)                                   # never its own neighbour
    nbr = np.lexsort((idx, de), axis=1)[:, :k]
    t = float(np.maximum(np.take_along_axis(rank, nbr, axis=1) - k, 0).sum())
    return 1.0 - (2.0 / ((n * k) * ((2.0 * n) - (3.0 * k) - 1.0))) * t


def compare_approx(a, b, eps):
    """raft::CompareApprox: cpp/tests/test_utils.h:31-45 (relative when diff > eps, else
    absolute).  Vectorised; returns a boolean array."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    diff = np.abs(a - b)
    m = np.maximum(np.abs(a), np.abs(b))
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(diff > eps, diff / m, diff)
    both_nan = np.isnan(a) & np.isnan(b)     # CompareApproxNaN, test_utils.h:47-63
    return (ratio <= eps) | both_nan


def match_approx(actual, expected, eps):
    ok = compare_approx(actual, expected, eps)
    if ok.all():
        return True, ""
    bad = np.argwhere(~ok)
    i = tuple(bad[0])
    return False, (f"{(~ok).sum()} mismatches of {ok.size}; first at {i}: "
                   f"actual={np.asarray(actual)[i]!r} expected={np.asarray(expected)[i]!r}")


def pack_minloc(val_f32: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """Host model of the packed min-loc key the multi-GPU exchange reduces with MIN
    (SURVEY.md 8(e)): high 32 bits = float bits remapped so that signed-integer order equals
    float order, low 32 bits = index.  int64 MIN == (min value, then smaller index)."""
    bits = np.asarray(val_f32, dtype=np.float32).view(np.int32).astype(np.int64)
    s = np.where(bits < 0, bits ^ 0x7FFFFFFF, bits)
    return (s << 32) | (np.asarray(idx).astype(np.int64) & 0xFFFFFFFF)


def unpack_minloc(key: np.ndarray):
    key = np.asarray(key, dtype=np.int64)
    idx = (key & 0xFFFFFFFF).astype(np.int32)
    s = (key >> 32).astype(np.int64)
    bits = np.where(s < 0, s ^ 0x7FFFFFFF, s).astype(np.int32)
    return bits.view(np.float32), idx


def make_blobs(n_rows, n_cols, n_clusters=5, cluster_std=1.0, box=(-10.0, 10.0), seed=1234,
               centers=None, dtype=np.float32):
    """Isotropic Gaussian blobs like raft::random::make_blobs
    (cpp/include/raft/random/make_blobs.cuh:124-140 defaults: 5 clusters, std 1, centre box
    [-10,10]).  Same distribution, not the same bit pattern (SURVEY.md row 11)."""
    rng = np.random.default_rng(seed)
    if centers is None:
        centers = rng.uniform(box[0], box[1], size=(n_clusters, n_cols))
    labels = rng.integers(0, centers.shape[0], size=n_rows)
    data = centers[labels] + cluster_std * rng.standard_normal((n_rows, n_cols))
    return data.astype(dtype), labels.astype(np.int32), centers
