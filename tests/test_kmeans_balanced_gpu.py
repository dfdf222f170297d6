"""Balanced k-means on the GPU (raft_b200.cluster.kmeans_balanced; include/raft_b200.h: b2d_kmeans_balanced_fit): the
returned centroids are the k-means update of the returned labels bit for bit, the labels and centroids match the numpy
model (tests/kmeans_balanced_ref.py) on separated blobs, balance and quality against plain k-means, determinism and
CUDA-graph replay, and the edges (tiny and maximal n_clusters, duplicates, k of 1 / 320 / 784, NaN rows)."""
import ctypes

import numpy as np
import pytest
import torch

import kmeans_balanced_ref as ref
import kmeans_ref
from raft_b200 import _lib
from raft_b200.cluster import KMeansParams, compute_new_centroids
from raft_b200.cluster import fit as km_fit
from raft_b200.cluster import kmeans_balanced as kb

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(a):
    return torch.as_tensor(a, device="cuda").cpu().numpy()


def fit_predict(x, nc, n_iters=20, seed=0):
    c, lab, sizes = kb.fit_predict(kb.KMeansBalancedParams(n_iters=n_iters, seed=seed), dev(x), nc)
    return host(c), host(lab), host(sizes)


def check_update(x, c, lab, sizes):
    """centroids == compute_new_centroids(x, centroids, labels) bit for bit; sizes == bincount(labels)"""
    nc = len(c)
    new = torch.empty((nc, x.shape[1]), dtype=torch.float32, device="cuda")
    compute_new_centroids(dev(x), dev(c), dev(lab.astype(np.int32)), new)
    assert host(new).tobytes() == c.tobytes()
    assert (sizes == np.bincount(lab[lab >= 0], minlength=nc)).all()
    assert np.isfinite(c).all()


@pytest.mark.parametrize("m,k,nc", [(3000, 16, 1), (3000, 16, 2), (3000, 16, 3), (5000, 32, 100), (20011, 64, 400),
                                    (4000, 1, 30), (6000, 320, 64), (3001, 784, 50), (777, 8, 777)])
def test_centroids_are_the_update_of_the_labels(m, k, nc):
    x, _, _ = kmeans_ref.blobs(m, k, max(1, nc // 3), seed=m + k, spread=0.5)
    c, lab, sizes = fit_predict(x, nc, 10, seed=3)
    check_update(x, c, lab, sizes)
    assert (lab >= 0).all() and (lab < nc).all()
    if nc == m:   # one row per cluster
        assert (sizes == 1).all()


@pytest.mark.parametrize("m,k,nc,n_iters,seed", [(3000, 4, 40, 6, 11), (5000, 8, 60, 10, 3), (4001, 16, 30, 20, 0)])
def test_matches_the_model(m, k, nc, n_iters, seed):
    """Uniform data, where the adjust step fires in every stage: the device draws the model's donors and takes its
    decisions, so labels and sizes are equal and centroids agree to 1e-5."""
    x = np.random.default_rng(seed).uniform(-1, 1, size=(m, k)).astype(np.float32)
    c, lab, sizes = fit_predict(x, nc, n_iters, seed=seed)
    rc, rlab, rsizes = ref.fit(x, nc, n_iters, seed=seed)
    assert (lab == rlab).all()
    assert (sizes == rsizes).all()
    np.testing.assert_allclose(c, rc, rtol=1e-5, atol=1e-5 * np.abs(rc).max())


@pytest.mark.parametrize("m,k,nc,n_iters", [(3000, 8, 12, 10), (10000, 32, 100, 20), (6007, 16, 49, 5)])
def test_close_to_the_model_on_separated_blobs(m, k, nc, n_iters):
    """One tight blob per cluster.  The stages can put two centroids on one blob for a while, and the rows on the
    boundary they draw through a blob are near-ties that fp32 and fp64 decide differently (measured agreement:
    0.9936-0.9990), so only 99 % of the labels are held to the model.  A cluster with the same rows on both sides has
    the same centroid to 1e-5, and at least 80 % of the clusters are such clusters."""
    x, _, _ = kmeans_ref.blobs(m, k, nc, seed=nc, spread=0.002)
    c, lab, sizes = fit_predict(x, nc, n_iters, seed=5)
    rc, rlab, rsizes = ref.fit(x, nc, n_iters, seed=5)
    assert (lab == rlab).mean() >= 0.99
    same = [j for j in range(nc) if sizes[j] == rsizes[j] and (np.flatnonzero(lab == j) == np.flatnonzero(rlab == j)).all()]
    assert len(same) >= 0.8 * nc, (len(same), nc)
    np.testing.assert_allclose(c[same], rc[same], rtol=1e-5, atol=1e-5 * np.abs(rc).max())


def spreads(sizes):
    avg = sizes.sum() / len(sizes)
    return sizes.min() / avg, sizes.max() / avg


@pytest.mark.parametrize("kind", ["uniform", "skewed"])
def test_balance(kind):
    """Thresholds from the model (tests/test_kmeans_balanced.py: [0.25, 1.7] of the average size at 4000 x 8 and 64
    clusters), here at 50000 x 16 and 256 clusters; the spreads of plain kmeans.fit are printed beside them."""
    rng = np.random.default_rng(1)
    m, k, nc = 50000, 16, 256
    if kind == "uniform":
        x = rng.uniform(-1, 1, size=(m, k)).astype(np.float32)
    else:
        big = rng.normal(0, 0.05, size=(m - m // 10, k))
        x = np.concatenate([big, rng.normal(0, 1.0, size=(m // 10, k)) + 4]).astype(np.float32)[rng.permutation(m)]
    c, lab, sizes = fit_predict(x, nc, 20, seed=0)
    lo, hi = spreads(sizes)
    o = km_fit(KMeansParams(n_clusters=nc, max_iter=20, tol=0.0, oversampling_factor=2.0), dev(x))
    plab, _ = kmeans_ref.assign(x, host(o.centroids))
    print("balanced min/avg %.3f max/avg %.3f | kmeans min/avg %.3f max/avg %.3f" %
          ((lo, hi) + spreads(np.bincount(plab, minlength=nc))))
    assert lo >= 0.25 and hi <= 1.7, (lo, hi)


@pytest.mark.parametrize("nc", [256, 1024])
def test_quality_against_kmeans(nc):
    """Inertia within 1.3 of a k-means||-seeded kmeans.fit with the same iteration budget (the model's factor on
    uniform and skewed data: 1.01-1.16)."""
    x, _, _ = kmeans_ref.blobs(100000, 32, nc // 2, seed=nc, spread=0.3)
    c, lab, sizes = fit_predict(x, nc, 20, seed=0)
    o = km_fit(KMeansParams(n_clusters=nc, max_iter=22, tol=0.0, oversampling_factor=2.0), dev(x))
    mine = kmeans_ref.cost(x, c)
    print("nc %d balanced inertia / kmeans inertia %.4f" % (nc, mine / o.inertia))
    assert mine < 1.3 * o.inertia


def test_deterministic_and_graph_replay():
    x, _, _ = kmeans_ref.blobs(60000, 128, 50, seed=21, spread=0.5)
    a, b = fit_predict(x, 300, 8, seed=2), fit_predict(x, 300, 8, seed=2)
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()
    L = _lib.lib()
    m, k, nc = x.shape[0], x.shape[1], 300
    xd = dev(x)
    c = torch.empty((nc, k), dtype=torch.float32, device="cuda")
    lab = torch.empty(m, dtype=torch.int32, device="cuda")
    sizes = torch.empty(nc, dtype=torch.int32, device="cuda")
    ws = torch.empty(L.b2d_kmeans_balanced_workspace_bytes(m, k, nc), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_kmeans_balanced_fit(ctypes.c_void_p(s.cuda_stream), nc, 8, 2, xd.data_ptr(), k, m, k,
                                             c.data_ptr(), lab.data_ptr(), sizes.data_ptr(), ws.data_ptr(), ws.numel()))
    c.zero_()
    lab.zero_()
    ws.fill_(0xFF)
    g.replay()
    torch.cuda.synchronize()
    assert c.cpu().numpy().tobytes() == a[0].tobytes()
    assert lab.cpu().numpy().tobytes() == a[1].tobytes()
    assert sizes.cpu().numpy().tobytes() == a[2].tobytes()


def test_fewer_distinct_rows_than_clusters():
    base = np.random.default_rng(3).normal(size=(7, 16)).astype(np.float32)
    x = base[np.arange(2000) % 7]
    c, lab, sizes = fit_predict(x, 50, 10)
    check_update(x, c, lab, sizes)
    assert len(np.unique(c, axis=0)) <= 50 and (sizes > 0).sum() >= 7


def test_nan_rows():
    x, _, _ = kmeans_ref.blobs(5003, 24, 10, seed=9, spread=0.1)
    bad = [0, 17, 2500, 5002]
    x[bad] = np.nan
    x[100, 3] = np.inf
    c, lab, sizes = fit_predict(x, 40, 10)
    assert (lab[bad + [100]] == -1).all() and (np.delete(lab, bad + [100]) >= 0).all()
    assert np.isfinite(c).all() and sizes.sum() == 5003 - 5
    check_update(x, c, lab, sizes)


def test_fit_and_predict():
    x, _, _ = kmeans_ref.blobs(8000, 16, 20, seed=4, spread=0.05)
    p = kb.KMeansBalancedParams(n_iters=10, seed=1)
    c = kb.fit(p, dev(x), 20)
    c2, lab, _ = kb.fit_predict(p, dev(x), 20)
    assert host(c).tobytes() == host(c2).tobytes()
    # the fit's labels are the assignment its last update used; predict assigns to the updated centroids
    pl = host(kb.predict(p, dev(x), c))
    assert (pl == host(lab)).mean() > 0.99 and (pl >= 0).all()
    out = torch.empty((20, 16), dtype=torch.float32, device="cuda")
    kb.fit(p, dev(x), centroids=out)
    assert out.cpu().numpy().tobytes() == host(c).tobytes()
