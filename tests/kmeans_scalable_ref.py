"""numpy model of the k-means|| seeding of raft_b200.cluster.init_scalable (include/raft_b200.h: b2d_kmeans_init_scalable)
and of greedy k-means++, in fp64.  The random numbers come from a numpy generator, not Philox, so the model reproduces
the law of the device's draws, not its bits; the GPU tests take their quality thresholds from runs of this model."""
import math

import numpy as np

import kmeans_ref

ROUNDS = 8


def sizes(m, nc, f):
    """(L, C): L rows per oversampling round, C = 1 + 8L candidates."""
    L = min(m, max(math.ceil(f * nc), math.ceil((nc - 1) / ROUNDS)))
    return L, 1 + ROUNDS * L


def es_draw(p, n, rng):
    """n rows without replacement with probability ~ p (Efraimidis-Spirakis: the n smallest ln(E) - ln(p), E ~ Exp(1));
    mass 0 gives +inf and a NaN mass NaN, ranked after +inf; ties to the smaller row."""
    with np.errstate(divide="ignore", invalid="ignore"):
        key = np.log(rng.exponential(size=len(p))) - np.log(p)
    key = np.where(p == 0, np.inf, key)
    key = np.where(np.isnan(key), np.inf, key)
    rank = np.where(np.isnan(p), 1, 0)
    return np.lexsort((np.arange(len(p)), key, rank))[:n]


def d2_to(x, c):
    return kmeans_ref.assign(x, c)[1]


def candidates(x, nc, f, w=None, seed=0):
    """(candidate row ids [C], candidate weights [C]) of the k-means|| rounds."""
    rng = np.random.default_rng(seed)
    x = np.asarray(x, np.float64)
    m = len(x)
    w = np.ones(m) if w is None else np.maximum(np.asarray(w, np.float64), 0.0)
    L, _ = sizes(m, nc, f)
    ids = list(es_draw(w, 1, rng))
    D = d2_to(x, x[ids])
    D[ids] = 0.0
    for _ in range(ROUNDS):
        new = es_draw(w * D, L, rng)
        ids += list(new)
        D = np.minimum(D, d2_to(x, x[new]))
        D[new] = 0.0
    ids = np.array(ids)
    lab, _ = kmeans_ref.assign(x, x[ids])
    W = np.bincount(lab, weights=w, minlength=len(ids))
    return ids, W


def greedy_plus_plus(x, nc, w=None, seed=0):
    """Greedy k-means++ with 2 + floor(ln nc) trials per round: centroids [nc, k]."""
    rng = np.random.default_rng(seed)
    x = np.asarray(x, np.float64)
    m = len(x)
    w = np.ones(m) if w is None else np.maximum(np.asarray(w, np.float64), 0.0)
    trials = 2 + int(math.floor(math.log(nc)))
    first = rng.choice(m, p=w / w.sum())
    chosen = [first]
    D = ((x - x[first]) ** 2).sum(1)
    for _ in range(1, nc):
        p = w * D
        tot = p.sum()
        cand = rng.choice(m, size=trials, p=p / tot) if tot > 0 else rng.choice(m, size=trials)
        pots = [(w * np.minimum(D, ((x - x[c]) ** 2).sum(1))).sum() for c in cand]
        best = cand[int(np.argmin(pots))]
        chosen.append(best)
        D = np.minimum(D, ((x - x[best]) ** 2).sum(1))
    return x[chosen].astype(np.float32)


def init_scalable(x, nc, f=2.0, w=None, seed=0):
    """k-means|| centroids [nc, k]: the candidates, greedy k-means++ on them with weights W, then Lloyd (max_iter 300,
    tol 1e-4) on them with weights W."""
    ids, W = candidates(x, nc, f, w, seed)
    cand = np.asarray(x, np.float32)[ids]
    c0 = greedy_plus_plus(cand, nc, W, seed + 1)
    c, _, _, _ = kmeans_ref.lloyd(cand, c0, 300, 1e-4, w=W.astype(np.float32))
    return c
