"""numpy model of raft_b200.cluster.kmeans_balanced (include/raft_b200.h: b2d_kmeans_balanced_fit): the three stages of
balanced EM, the fine allocation and the adjust step with the device's Philox4x32-10 draws.  Distances and sums are fp64;
centroids are rounded to fp32 after every update and every adjust, as on the device, so on well-separated data the model
takes the same decisions and returns the same labels."""
import math

import numpy as np

import kmeans_ref

MESO, FINE, FINAL = 0, 1, 2
MAX_WEIGHT = 7
_M = 0xffffffff


def groups(nc):
    """G = min(n_clusters, max(1, round(sqrt(n_clusters)))) mesoclusters (sqrt of an integer is never a half)."""
    return min(nc, max(1, int(round(math.sqrt(nc)))))


def philox4x32_10(ctr, key):
    """curand_Philox4x32_10: ten rounds on the counter (4 words) with the key (2 words) bumped between rounds."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & _M, (k1 + 0xBB67AE85) & _M
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & _M, p1 & _M, ((p0 >> 32) ^ c3 ^ k1) & _M, p0 & _M
    return c0, c1, c2, c3


def draw(seed, stage, it, j, R):
    """The donor position of centroid j in [0, R): floor(((w0 << 32) | w1) R / 2^64), Philox counter (j, it, stage, 0)
    and key (seed low, seed high)."""
    w = philox4x32_10((j & _M, it & _M, stage, 0), (seed & _M, (seed >> 32) & _M))
    return ((w[0] << 32 | w[1]) * R) >> 64


def allocate(S, nc):
    """Fine clusters per mesocluster of sizes S: floor(nc S_g / R) plus one for the largest remainders (ties: lower g);
    then each non-empty mesocluster with none takes one from the largest a / S holding at least two (ties: lower g)."""
    S = [int(s) for s in S]
    G, R = len(S), sum(S)
    if R == 0:
        return [nc] + [0] * (G - 1)
    a = [nc * s // R for s in S]
    left = nc - sum(a)
    for g in sorted(range(G), key=lambda g: (-(nc * S[g] % R), g))[:left]:
        a[g] += 1
    for g in range(G):
        if a[g] > 0 or S[g] == 0:
            continue
        best = -1
        for h in range(G):
            if a[h] >= 2 and (best < 0 or a[h] * S[best] > a[best] * S[h]):
                best = h
        if best < 0:
            break
        a[best] -= 1
        a[g] = 1
    return a


def _em(x, probs, c, iters, seed, stage):
    """Balanced EM on the problems probs = [(rows in problem order, first centroid, centroid count)]: centroids c
    [nc, k] float32 (in place) and the labels [m] of the last assignment (-1: in no problem)."""
    m = len(x)
    for it in range(iters):
        lab = np.full(m, -1, np.int64)
        for rows, c0, C in probs:
            if len(rows) and C:
                lab[rows] = c0 + kmeans_ref.assign(x[rows], c[c0:c0 + C])[0]
        c[:], _ = kmeans_ref.update(x, lab, c)
        if it + 1 == iters:
            return lab
        size = np.bincount(lab[lab >= 0], minlength=len(c))
        for rows, c0, C in probs:
            R = len(rows)
            for j in range(c0, c0 + C):
                s = int(size[j])
                if R == 0 or not 4 * s * C < R:
                    continue
                d = rows[draw(seed, stage, it, j, R)]
                if lab[d] < 0 or size[lab[d]] * C < R:
                    continue
                w = float(min(s, MAX_WEIGHT))
                c[j] = ((w * c[j].astype(np.float64) + x[d].astype(np.float64)) / (w + 1.0)).astype(np.float32)
    return lab


def _strided(x, rows, C):
    R = len(rows)
    if R == 0:
        return np.zeros((C, x.shape[1]), np.float32)
    return x[rows[(np.arange(C) * R) // C]].astype(np.float32)


def fit(x, nc, n_iters=20, seed=0, stages=False):
    """(centroids float32 [nc, k], labels int [m], sizes int [nc]); with stages also the mesocluster labels, the
    allocation and the fine stage's centroids and labels (in row order)."""
    x = np.asarray(x, np.float32)
    valid = np.flatnonzero(np.isfinite(x).all(1))
    G = groups(nc)
    cm = _strided(x, valid, G)
    meso = _em(x, [(valid, 0, G)], cm, n_iters, seed, MESO)
    S = np.bincount(meso[meso >= 0], minlength=G)
    a = allocate(S, nc)
    F = np.concatenate([[0], np.cumsum(a)])
    c = np.zeros((nc, x.shape[1]), np.float32)
    probs = []
    for g in range(G):
        rows = np.flatnonzero(meso == g)
        c[F[g]:F[g + 1]] = _strided(x, rows, a[g])
        probs.append((rows, int(F[g]), a[g]))
    fine = _em(x, probs, c, n_iters, seed, FINE)
    cf = c.copy()
    lab = _em(x, [(valid, 0, nc)], c, max(n_iters // 10, 2), seed, FINAL)
    sizes = np.bincount(lab[lab >= 0], minlength=nc)
    if stages:
        return c, lab, sizes, dict(meso=meso, alloc=a, fine_centroids=cf, fine_labels=fine)
    return c, lab, sizes
