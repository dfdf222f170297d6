"""kmeans on the GPU against the fp64 reference (tests/kmeans_ref.py), the fused L2 arg-min, and itself (determinism,
CUDA-graph capture)."""
import ctypes

import numpy as np
import pytest
import torch

import kmeans_ref
from raft_b200 import _lib
from raft_b200.cluster import KMeansParams, cluster_cost, compute_new_centroids, fit, init_plus_plus, predict
from raft_b200.distance import fused_l2_nn

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(a):
    return torch.as_tensor(a, device="cuda").cpu().numpy()


def ulps(a, b):
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def gpu_update(x, labels, old, w=None):
    nc, k = old.shape
    new = torch.empty((nc, k), dtype=torch.float32, device="cuda")
    wpc = torch.empty(nc, dtype=torch.float32, device="cuda")
    compute_new_centroids(dev(x), dev(old), dev(labels.astype(np.int32)), new,
                          sample_weights=None if w is None else dev(w), weight_per_cluster=wpc)
    return new.cpu().numpy(), wpc.cpu().numpy()


def check_update(x, labels, old, w=None):
    got, wpc = gpu_update(x, labels, old, w)
    ref, rw = kmeans_ref.update(x, labels, old, w)
    assert ulps(got, ref).max() <= 1
    W = np.zeros(old.shape[0])
    ok = (labels >= 0) & (labels < old.shape[0])
    np.add.at(W, labels[ok], (np.ones(len(x)) if w is None else w.astype(np.float64))[ok])
    empty = W == 0
    assert (got[empty].view(np.int32) == old[empty].view(np.int32)).all()   # bits kept
    np.testing.assert_array_equal(wpc, rw)


@pytest.mark.parametrize("k", [1, 3, 32, 128, 129, 320, 784])
@pytest.mark.parametrize("weighted", [False, True])
def test_update_matches_fp64(k, weighted):
    rng = np.random.default_rng(k)
    m, nc = 5000 + 37, 50            # m not a multiple of the 2048-row sort block nor of the 256-row chunk
    x = rng.normal(size=(m, k)).astype(np.float32) * 3 + 1
    labels = rng.integers(0, nc - 5, size=m)           # clusters nc-5.. are empty
    labels[::97] = -3                                   # out of range: skipped
    labels[5::101] = nc + 7
    old = rng.normal(size=(nc, k)).astype(np.float32)
    w = rng.uniform(0.1, 2.0, size=m).astype(np.float32) if weighted else None
    if weighted:
        w[labels == 3] = 0.0                            # a zero-weight cluster keeps its bits too
    check_update(x, labels, old, w)


@pytest.mark.parametrize("nc", [1, 100000])
def test_update_cluster_counts(nc):
    rng = np.random.default_rng(nc)
    m, k = 200003, 16
    x = rng.normal(size=(m, k)).astype(np.float32)
    labels = rng.integers(0, nc, size=m)
    check_update(x, labels, rng.normal(size=(nc, k)).astype(np.float32))


def test_update_above_the_histogram_cap():
    # 10^5 clusters x ceil(10^6 / 2048) blocks exceeds the 2^24-word histogram: each sort block then spans several
    # 2048-row sub-blocks, whose cursors carry over from one sub-block to the next
    rng = np.random.default_rng(12)
    m, k, nc = 10 ** 6, 4, 10 ** 5
    assert nc * -(-m // 2048) > 2 ** 24
    x = rng.normal(size=(m, k)).astype(np.float32)
    labels = rng.integers(0, nc, size=m)
    labels[::1000] = -1
    check_update(x, labels, rng.normal(size=(nc, k)).astype(np.float32))


def test_update_giant_cluster_next_to_singletons():
    rng = np.random.default_rng(7)
    m, k, nc = 10 ** 6 + 300, 8, 301
    x = rng.normal(size=(m, k)).astype(np.float32) + 100
    labels = np.zeros(m, np.int64)
    labels[rng.choice(m, 300, replace=False)] = np.arange(1, 301)
    check_update(x, labels, rng.normal(size=(nc, k)).astype(np.float32), rng.uniform(0.5, 1.5, m).astype(np.float32))


def near_ties_only(x, c, labels, ref_labels, ref_d):
    """Every label that differs from the exact fp64 arg-min is a provable near-tie (|dd| <= 1e-5 d); returns the count."""
    bad = labels != ref_labels
    if bad.any():
        dg = ((x[bad].astype(np.float64) - c[labels[bad]].astype(np.float64)) ** 2).sum(1)
        assert (np.abs(dg - ref_d[bad]) <= 1e-5 * np.maximum(ref_d[bad], 1e-30)).all()
    return int(bad.sum())


@pytest.mark.parametrize("k,nc", [(32, 17), (128, 256), (320, 1000), (784, 257)])
def test_predict_matches_fused_l2_nn(k, nc):
    x, _, _ = kmeans_ref.blobs(20000, k, nc, seed=k)
    c = x[np.random.default_rng(1).choice(len(x), nc, replace=False)] + 0.01
    _lib.check(_lib.lib().b2d_set_option(b"nn_screen", 0))
    try:
        idx, _ = fused_l2_nn(dev(x), dev(c), sqrt=False)
    finally:
        _lib.check(_lib.lib().b2d_set_option(b"nn_screen", 1))
    labels, inertia = predict(KMeansParams(n_clusters=nc), dev(x), dev(c))
    labels = host(labels)
    assert (labels == idx.cpu().numpy()).all()
    rl, rd = kmeans_ref.assign(x, c)
    assert near_ties_only(x, c, labels, rl, rd) <= 10
    assert abs(inertia - rd.sum()) <= 1e-4 * rd.sum()
    assert abs(cluster_cost(dev(x), dev(c)) - inertia) == 0


@pytest.mark.parametrize("nc,k", [(2, 32), (17, 128), (256, 320), (257, 784), (1000, 128)])
@pytest.mark.parametrize("mode", ["tol0", "tol", "inertia_check"])
def test_fit_array_matches_reference(nc, k, mode):
    x, _, _ = kmeans_ref.blobs(30000, k, nc, seed=nc + k, spread=0.3)
    c0 = x[np.random.default_rng(nc).choice(len(x), nc, replace=False)]
    tol, max_iter, ic = {"tol0": (0.0, 8, False), "tol": (1e-2, 100, False), "inertia_check": (1e-3, 100, True)}[mode]
    ref_c, ref_lab, ref_in, ref_it = kmeans_ref.lloyd(x, c0, max_iter, tol, inertia_check=ic)
    c = dev(c0)
    out = fit(KMeansParams(n_clusters=nc, max_iter=max_iter, tol=tol, init_method="Array", inertia_check=ic), dev(x), c)
    assert out.n_iter == ref_it
    assert ulps(c.cpu().numpy(), ref_c).max() <= 1
    labels, _ = predict(KMeansParams(n_clusters=nc), dev(x), c)
    # the final labels equal the reference's, except provable near-ties under the reference's centroids
    _, ref_d = kmeans_ref.assign(x, ref_c)
    assert near_ties_only(x, ref_c, host(labels), ref_lab, ref_d) <= 10
    assert abs(out.inertia - ref_in) <= 1e-4 * ref_in


def test_fit_edge_cases():
    x, _, _ = kmeans_ref.blobs(4000, 16, 4, seed=3)
    # a centroid far from every row stays put (its cluster is empty)
    c0 = np.concatenate([x[:3], np.full((1, 16), 1e4, np.float32)])
    c = dev(c0)
    fit(KMeansParams(n_clusters=4, max_iter=5, tol=0.0, init_method="Array"), dev(x), c)
    assert (c.cpu().numpy()[3] == c0[3]).all()
    # n_clusters == m: every row its own centroid, inertia 0
    xs = x[:64].copy()
    out = fit(KMeansParams(n_clusters=64, max_iter=3, init_method="Array"), dev(xs), dev(xs))
    assert out.inertia == 0.0 and out.n_iter == 1
    # NaN rows: no label, NaN inertia, no fault
    xn = x.copy()
    xn[[5, 700]] = np.nan
    c = dev(x[:4])
    out = fit(KMeansParams(n_clusters=4, max_iter=5, tol=0.0, init_method="Array"), dev(xn), c)
    assert np.isnan(out.inertia) and np.isfinite(c.cpu().numpy()).all()
    labels, _ = predict(KMeansParams(n_clusters=4), dev(xn), c)
    assert (host(labels)[[5, 700]] == -1).all()
    # negative weights: NaN inertia
    w = np.ones(len(x), np.float32)
    w[9] = -1
    assert np.isnan(fit(KMeansParams(n_clusters=4, max_iter=2, init_method="Array"), dev(x), dev(x[:4]),
                        sample_weights=dev(w)).inertia)


def test_fit_weighted_matches_reference():
    x, _, _ = kmeans_ref.blobs(20000, 64, 20, seed=11, spread=0.3)
    w = np.random.default_rng(2).uniform(0.2, 3.0, len(x)).astype(np.float32)
    c0 = x[:20]
    ref_c, _, ref_in, ref_it = kmeans_ref.lloyd(x, c0, 30, 1e-4, w=w)
    c = dev(c0)
    out = fit(KMeansParams(n_clusters=20, max_iter=30, tol=1e-4, init_method="Array"), dev(x), c, sample_weights=dev(w))
    assert out.n_iter == ref_it and ulps(c.cpu().numpy(), ref_c).max() <= 1
    assert abs(out.inertia - ref_in) <= 1e-4 * ref_in


def rows_of(c, x):
    xs = {r.tobytes(): i for i, r in enumerate(x)}
    return [xs.get(r.tobytes(), -1) for r in c]


def test_init_plus_plus():
    x, lab, _ = kmeans_ref.blobs(50000, 32, 12, seed=5, spread=0.01)
    a = host(init_plus_plus(dev(x), n_clusters=12, seed=3))
    b = host(init_plus_plus(dev(x), n_clusters=12, seed=3))
    d = host(init_plus_plus(dev(x), n_clusters=12, seed=4))
    assert a.tobytes() == b.tobytes() and a.tobytes() != d.tobytes()
    r = rows_of(a, x)
    assert min(r) >= 0
    assert sorted(lab[r]) == list(range(12))                       # one seed per blob


def test_init_plus_plus_never_draws_zero_weight_or_duplicates():
    rng = np.random.default_rng(8)
    m, k, nc = 3000, 8, 40
    x = rng.normal(size=(m, k)).astype(np.float32)
    x[1000:2000] = x[0]                                           # duplicates of row 0
    w = np.ones(m, np.float32)
    w[2000:] = 0.0                                                # never drawn
    xd, wd = dev(x), dev(w)
    c = torch.empty((nc, k), dtype=torch.float32, device="cuda")
    L = _lib.lib()
    ws = torch.empty(L.b2d_kmeans_workspace_bytes(m, k, nc), dtype=torch.uint8, device="cuda")
    for seed in range(5):
        _lib.check(L.b2d_kmeans_init_plus_plus(None, xd.data_ptr(), k, wd.data_ptr(), m, k, nc, seed, c.data_ptr(),
                                               ws.data_ptr(), ws.numel()))
        torch.cuda.synchronize()
        r = np.array(rows_of(c.cpu().numpy(), x))
        assert (r >= 0).all() and (r < 2000).all()
        assert len(np.unique(c.cpu().numpy(), axis=0)) == nc       # a duplicate of a chosen row is never drawn


def test_random_init_and_n_init():
    x, _, _ = kmeans_ref.blobs(20000, 16, 8, seed=9, spread=0.2)
    out = fit(KMeansParams(n_clusters=64, max_iter=0, init_method="Random", seed=5), dev(x))
    r = rows_of(host(out.centroids), x)
    assert min(r) >= 0 and len(set(r)) == 64
    runs = [fit(KMeansParams(n_clusters=8, max_iter=20, init_method="KMeansPlusPlus", seed=10 + s), dev(x)) for s in range(3)]
    best = min(range(3), key=lambda s: (runs[s].inertia, s))
    out = fit(KMeansParams(n_clusters=8, max_iter=20, init_method="KMeansPlusPlus", seed=10, n_init=3), dev(x))
    assert host(out.centroids).tobytes() == host(runs[best].centroids).tobytes()
    assert out.inertia == runs[best].inertia and out.n_iter == runs[best].n_iter


def test_determinism_and_graph_capture():
    x, _, _ = kmeans_ref.blobs(100000, 128, 64, seed=21, spread=0.5)
    xd = dev(x)
    p = KMeansParams(n_clusters=64, max_iter=15, tol=0.0, init_method="KMeansPlusPlus", seed=2)
    a, b = fit(p, xd), fit(p, xd)
    assert host(a.centroids).tobytes() == host(b.centroids).tobytes()
    assert a.inertia == b.inertia and a.n_iter == b.n_iter == 15
    L = _lib.lib()
    m, k, nc = x.shape[0], x.shape[1], 64
    c = torch.empty((nc, k), dtype=torch.float32, device="cuda")
    inertia = torch.empty(1, dtype=torch.float64, device="cuda")
    n_iter = torch.empty(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(L.b2d_kmeans_workspace_bytes(m, k, nc), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_kmeans_fit(ctypes.c_void_p(s.cuda_stream), nc, 15, 0.0, 0, 1, 2, 0, xd.data_ptr(), k, None, m, k,
                                    c.data_ptr(), inertia.data_ptr(), n_iter.data_ptr(), ws.data_ptr(), ws.numel()))
    c.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert c.cpu().numpy().tobytes() == host(a.centroids).tobytes()
    assert inertia.item() == a.inertia and n_iter.item() == 15
