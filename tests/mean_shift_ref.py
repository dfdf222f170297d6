"""fp64 numpy model of b2d_mean_shift_fit (include/raft_b200.h).  The neighbourhood test is passed in, so the model runs
on sklearn's exact distances (``exact_within``) or on the engine's squared distances.

  within(P, Q) -> bool [len(P), len(Q)]: row q of Q is within h of point p
  dist2(P, Q)  -> float [len(P), len(Q)]: the squared distances the labels are decided on
"""
import numpy as np


def exact_d2(P, Q):
    P = np.asarray(P, np.float64)
    Q = np.asarray(Q, np.float64)
    d2 = (P * P).sum(1)[:, None] + (Q * Q).sum(1)[None, :] - 2.0 * (P @ Q.T)
    return np.maximum(d2, 0.0)


def exact_within(h):
    return lambda P, Q: np.sqrt(exact_d2(P, Q)) <= h


def scale_exponent(a):
    """prep.cuh scale_exponent: the e that puts a > 0 into [2^14, 2^15), clamped to [-100, 100]; 0 for 0 or >= 3e38"""
    if not 0.0 < a < 3.0e38:
        return 0
    return int(np.clip(15 - np.frexp(a)[1], -100, 100))


def prep_scales(X):
    """The exponents the operand preparation (prep.cuh) gives the data rows of X [n, d] (fp32): (E, M, svec, own) with
    M the largest |element| of the rows whose maximum is finite (a NaN element is skipped), E = scale_exponent(M),
    own[j] when row j took its own exponent e_j and svec[j] = 2^(E - e_j) (1 for the other rows).  The neighbour sums
    multiply row j by fp16(svec[j]): rows with svec[j] < 2^-24 (fp16 rounds it to 0) are left out of the sums."""
    a = np.abs(np.asarray(X, np.float32).astype(np.float64))
    amax = np.where(np.isnan(a), 0.0, a).max(1)
    valid = (amax > 0) & (amax < 3.0e38)
    M = float(amax[valid].max()) if valid.any() else 0.0
    E = scale_exponent(M)
    own = valid & (amax * 2.0 ** E < 8.0)
    svec = np.ones(len(a))
    for j in np.flatnonzero(own):
        svec[j] = 2.0 ** (E - max(E, min(scale_exponent(amax[j]), E + 120)))
    return E, M, svec, own


def ordered_bits(v):
    """the fp32 order of v as int64, -0 before +0"""
    b = np.asarray(v, np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, b ^ 0x7FFFFFFF, b)


def bin_seeds(X, h, min_bin_freq=1):
    """sklearn's get_bin_seeds: bins rint(x / h) (fp64, ties to even), the bins with >= min_bin_freq rows at
    fp32(bin) * fp32(h) in order of their first row; the rows themselves when every row is a seed"""
    X = np.asarray(X, np.float32)
    bins = np.rint(X.astype(np.float64) / h) + 0.0
    _, first, counts = np.unique(bins, axis=0, return_index=True, return_counts=True)
    keep = np.sort(first[counts >= min_bin_freq])
    if len(keep) == len(X):
        return X.copy()
    return bins[keep].astype(np.float32) * np.float32(h)


def mean_shift(X, h, within, dist2, seeds=None, bin_seeding=False, min_bin_freq=1, cluster_all=True, max_iter=300, h2=None,
               trace=None):
    """(centers fp32 [K, d], labels int [n], n_iter); raises ValueError when no seed has a neighbour.  h2: the squared
    radius of cluster_all=False (default fp32(h * h)).  trace: a list that receives every shift the stop rule tests."""
    X = np.asarray(X, np.float32)
    Xd = X.astype(np.float64)
    if seeds is not None:
        S = np.asarray(seeds, np.float32)
    elif bin_seeding:
        S = bin_seeds(X, h, min_bin_freq)
    else:
        S = X.copy()
    means = S.copy()
    s = len(S)
    state = np.zeros(s, int)   # 0 active, 1 stopped, 2 dropped
    iters = np.zeros(s, int)
    inten = np.zeros(s, int)
    thr = 1e-3 * h
    while (state == 0).any():
        act = np.flatnonzero(state == 0)
        A = within(means[act], X)
        for r, i in enumerate(act):
            nb = A[r]
            cnt = int(nb.sum())
            if cnt == 0:
                state[i] = 2
                continue
            new = (Xd[nb].sum(0) / cnt).astype(np.float32)
            shift = np.linalg.norm(new.astype(np.float64) - means[i].astype(np.float64))
            means[i], inten[i] = new, cnt
            if trace is not None:
                trace.append(shift)
            if shift <= thr or iters[i] == max_iter:
                state[i] = 1
            else:
                iters[i] += 1
    n_iter = int(iters.max()) if s else 0
    cand = {}
    for i in np.flatnonzero(state == 1):
        key = means[i].tobytes()
        cand[key] = max(cand.get(key, 0), int(inten[i]))
    if not cand:
        raise ValueError("No point was within bandwidth of any seed")
    items = [(c, np.frombuffer(k, np.float32)) for k, c in cand.items()]
    items.sort(key=lambda t: (t[0], tuple(ordered_bits(t[1]))), reverse=True)
    C = np.stack([m for _, m in items])
    W = within(C, C)
    W = W | W.T
    suppressed = np.zeros(len(C), bool)
    kept = []
    for i in range(len(C)):
        if suppressed[i]:
            continue
        kept.append(i)
        suppressed |= W[i]
    centers = C[kept]
    D = dist2(X, centers)
    labels = D.argmin(1)   # first minimum: ties to the smaller index
    if not cluster_all:
        lim = np.float32(h * h) if h2 is None else h2
        labels = np.where(D[np.arange(len(X)), labels] <= lim, labels, -1)
    return centers, labels, n_iter
