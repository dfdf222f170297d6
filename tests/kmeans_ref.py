"""fp64 reference of raft_b200.cluster.kmeans: Lloyd's iterations whose centroids are rounded to fp32 after every
update, so the reference takes the same assignment decisions as the device."""
import numpy as np


def assign(x, c):
    """(labels, squared distances) of the nearest centroid in fp64, ties to the smaller index."""
    x = np.asarray(x, np.float64)
    c = np.asarray(c, np.float64)
    d = (x * x).sum(1)[:, None] - 2.0 * x @ c.T + (c * c).sum(1)[None, :]
    d = np.maximum(d, 0.0)
    lab = np.argmin(d, axis=1)
    return lab, d[np.arange(len(x)), lab]


def update(x, labels, old, w=None):
    """(new centroids float32, weight per cluster float32): fp64 weighted means rounded once; a cluster of zero weight
    keeps its old centroid; labels outside [0, n_clusters) are skipped."""
    x = np.asarray(x, np.float64)
    nc = old.shape[0]
    w = np.ones(len(x)) if w is None else np.asarray(w, np.float64)
    ok = (labels >= 0) & (labels < nc)
    s = np.zeros((nc, x.shape[1]))
    W = np.zeros(nc)
    np.add.at(s, labels[ok], w[ok, None] * x[ok])
    np.add.at(W, labels[ok], w[ok])
    new = old.astype(np.float32).copy()
    nz = W != 0
    new[nz] = (s[nz] / W[nz, None]).astype(np.float32)
    return new, W.astype(np.float32)


def normalize(w, m):
    """Weights scaled to sum to m, as the fp32 product the device forms."""
    w = np.asarray(w, np.float32)
    return w * np.float32(m / w.astype(np.float64).sum())


def cost(x, c, w=None):
    _, d = assign(x, c)
    return float(d.sum() if w is None else (np.asarray(w, np.float64) * d).sum())


def lloyd(x, c0, max_iter, tol, w=None, inertia_check=False):
    """(centroids, labels of the returned centroids, inertia, n_iter) of the device's loop."""
    c = np.asarray(c0, np.float32).copy()
    wn = None if w is None else normalize(w, len(x))
    prior, n_iter = 0.0, 0
    for it in range(1, max_iter + 1):
        lab, d = assign(x, c)
        inertia = float(d.sum() if wn is None else (wn.astype(np.float64) * d).sum())
        new, _ = update(x, lab, c, wn)
        shift = float(((new.astype(np.float64) - c.astype(np.float64)) ** 2).sum())
        c = new
        n_iter = it
        done = shift < tol or (inertia_check and it > 1 and inertia / prior > 1.0 - tol)
        prior = inertia
        if done:
            break
    lab, d = assign(x, c)
    inertia = float(d.sum() if wn is None else (wn.astype(np.float64) * d).sum())
    return c, lab, inertia, n_iter


def blobs(m, k, n_centers, seed, spread=0.05, scale=10.0):
    rng = np.random.default_rng(seed)
    centers = rng.uniform(-scale, scale, size=(n_centers, k))
    lab = rng.integers(0, n_centers, size=m)
    lab[:n_centers] = np.arange(n_centers)
    x = centers[lab] + rng.normal(scale=spread * scale, size=(m, k))
    return x.astype(np.float32), lab, centers.astype(np.float32)
