"""fp64 reference of masked_l2_nn (raft::distance::masked_l2_nn), shared by the CPU and GPU tests: the distances in
blocks of rows of y like oracle.fused_l2_nn, non-adjacent pairs excluded, ties to the smaller index, and the value of a
row without any candidate that the library writes ({0x7fffffff, FLT_MAX}).  NaN distances (NaN rows, inf - inf) are no
candidates, as in the library's arg-min: a row whose every adjacent distance is NaN keeps that value."""
import numpy as np

NO_CANDIDATE = 0x7FFFFFFF
FLT_MAX = float(np.finfo(np.float32).max)


def column_groups(group_idxs, n):
    """[n] group of every row of y, -1 for the rows at or after the end of the last group."""
    gi = np.asarray(group_idxs, dtype=np.int64)
    grp = np.full(n, -1, dtype=np.int64)
    lo = 0
    for g, hi in enumerate(gi):
        grp[lo:hi] = g
        lo = hi
    return grp


def masked_l2_nn(x, y, adj, group_idxs, sqrt=False, block=4096):
    """Returns (idx int32 [m], val fp64 [m])."""
    x64 = np.ascontiguousarray(x, dtype=np.float64)
    y64 = np.ascontiguousarray(y, dtype=np.float64)
    adj = np.asarray(adj) != 0
    m, n = x64.shape[0], y64.shape[0]
    grp = column_groups(group_idxs, n)
    best_v = np.full(m, np.inf)
    best_i = np.full(m, NO_CANDIDATE, dtype=np.int64)
    xx = (x64 * x64).sum(1)
    for j0 in range(0, n, block):
        yb = y64[j0:j0 + block]
        gb = grp[j0:j0 + block]
        d = np.maximum(xx[:, None] + (yb * yb).sum(1)[None, :] - 2.0 * (x64 @ yb.T), 0.0)
        ok = (gb >= 0)[None, :] & adj[:, np.maximum(gb, 0)] if adj.shape[1] else np.zeros(d.shape, bool)
        d = np.where(ok & ~np.isnan(d), d, np.inf)     # a NaN distance never wins (np.argmin would pick it)
        loc = np.argmin(d, axis=1)
        v = d[np.arange(m), loc]
        upd = v < best_v                     # strict: the earlier (smaller) index wins ties
        best_v = np.where(upd, v, best_v)
        best_i = np.where(upd, loc + j0, best_i)
    none = ~np.isfinite(best_v)
    if sqrt:
        best_v = np.sqrt(best_v)
    best_v[none] = FLT_MAX
    return best_i.astype(np.int32), best_v


def tile_classes(adj, group_idxs, m, n):
    """numpy restatement of masked_tile_class: [ceil(m/64), ceil(n/128)] of 0 NONE / 1 ALL / 2 PARTIAL."""
    adj = np.asarray(adj) != 0
    grp = column_groups(group_idxs, n)
    S, H = (m + 63) // 64, (n + 127) // 128
    out = np.zeros((S, H), dtype=np.int64)
    for s in range(S):
        a = adj[64 * s:64 * s + 64]
        for h in range(H):
            g = grp[128 * h:128 * h + 128]
            ok = (g >= 0)[None, :] & a[:, np.maximum(g, 0)] if adj.shape[1] else np.zeros((a.shape[0], len(g)), bool)
            out[s, h] = 0 if not ok.any() else (1 if ok.all() else 2)
    return out
