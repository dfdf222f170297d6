"""k-means|| on the GPU: the candidate set and its weights against the fused L2 arg-min and the centroid update, the law
of the draws, recovery of separated blobs, quality against greedy k-means++ with thresholds from runs of the numpy model
(tests/kmeans_scalable_ref.py), the fit (n_init, CUDA-graph capture, weights, routing) and edge cases."""
import ctypes

import numpy as np
import pytest
import torch

import kmeans_ref
import kmeans_scalable_ref as ref
from raft_b200 import _lib
from raft_b200.cluster import KMeansParams, cluster_cost, compute_new_centroids, fit, init_plus_plus, init_scalable
from raft_b200.distance import fused_l2_nn

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(a):
    return torch.as_tensor(a, device="cuda").cpu().numpy()


def candidates(x, nc, f=2.0, seed=0, w=None):
    c, rows, wts = init_scalable(dev(x), n_clusters=nc, oversampling_factor=f, seed=seed,
                                 sample_weights=None if w is None else dev(w), return_candidates=True)
    return host(c), host(rows), host(wts)


def reference_weights(x, rows, w=None):
    """weight_per_cluster of compute_new_centroids over the labels of the unscreened fused_l2_nn against x[rows]"""
    cand = x[rows]
    _lib.check(_lib.lib().b2d_set_option(b"nn_screen", 0))
    try:
        idx, _ = fused_l2_nn(dev(x), dev(cand), sqrt=False)
    finally:
        _lib.check(_lib.lib().b2d_set_option(b"nn_screen", 1))
    new = torch.empty(cand.shape, dtype=torch.float32, device="cuda")
    wpc = torch.empty(len(rows), dtype=torch.float32, device="cuda")
    compute_new_centroids(dev(x), dev(cand), idx.to(torch.int32).contiguous(), new,
                          sample_weights=None if w is None else dev(w), weight_per_cluster=wpc)
    return wpc.cpu().numpy()


@pytest.mark.parametrize("m,k,nc,f", [(20000, 16, 10, 2.0), (50000, 128, 300, 0.5), (7000, 33, 64, 0.01)])
def test_candidates_and_weights(m, k, nc, f):
    x, _, _ = kmeans_ref.blobs(m, k, nc, seed=m + k, spread=0.3)
    c, rows, wts = candidates(x, nc, f, seed=3)
    L, C = ref.sizes(m, nc, f)
    assert len(rows) == C and len(wts) == C and c.shape == (nc, k) and np.isfinite(c).all()
    assert rows.min() >= 0 and rows.max() < m
    assert len(np.unique(rows)) == C                                  # rows with mass remain: all distinct
    assert wts.tobytes() == reference_weights(x, rows).tobytes()
    assert wts.astype(np.float64).sum() == m                          # unit weights: every row counted once
    c2, rows2, wts2 = candidates(x, nc, f, seed=3)
    assert rows2.tobytes() == rows.tobytes() and wts2.tobytes() == wts.tobytes() and c2.tobytes() == c.tobytes()
    assert candidates(x, nc, f, seed=4)[1].tobytes() != rows.tobytes()


def test_zero_weight_and_nan_rows_are_not_candidates():
    rng = np.random.default_rng(8)
    m, k, nc = 6000, 8, 40
    x = rng.normal(size=(m, k)).astype(np.float32)
    x[100:110] = np.nan
    w = rng.uniform(0.5, 2.0, m).astype(np.float32)
    w[3000:4000] = 0.0
    for seed in range(3):
        c, rows, wts = candidates(x, nc, 2.0, seed=seed, w=w)
        assert len(np.unique(rows)) == len(rows)
        assert not ((rows >= 3000) & (rows < 4000)).any()
        assert not ((rows >= 100) & (rows < 110)).any()
        assert np.isfinite(c).all()
    xc = x.copy()
    xc[100:110] = 0.0
    c, rows, wts = candidates(xc, nc, 2.0, seed=1, w=w)
    assert not ((rows >= 3000) & (rows < 4000)).any()
    assert wts.tobytes() == reference_weights(xc, rows, w).tobytes()


def chi2(obs, exp):
    keep = exp > 0
    assert obs[~keep].sum() == 0
    return float(((obs[keep] - exp[keep]) ** 2 / exp[keep]).sum())


def test_sampling_law():
    """16 rows, n_clusters = 1, f = 1 (L = 1): candidate 0 ~ w, candidate 1 given candidate 0 ~ w D^2.  A fixed seed
    range, so the test is deterministic; the bound is the 0.999 quantile of chi-square with 15 degrees of freedom."""
    rng = np.random.default_rng(2)
    m, k = 16, 3
    x = rng.normal(size=(m, k)).astype(np.float32)
    w = rng.uniform(1.0, 3.0, m).astype(np.float32)
    xd, wd = dev(x), dev(w)
    n = 1200
    first = np.zeros(m)
    second = np.zeros(m)
    exp2 = np.zeros(m)
    x64 = x.astype(np.float64)
    for seed in range(n):
        _, rows, _ = init_scalable(xd, n_clusters=1, oversampling_factor=1.0, seed=seed, sample_weights=wd,
                                   return_candidates=True)
        rows = host(rows)
        assert len(rows) == 9
        first[rows[0]] += 1
        second[rows[1]] += 1
        p = w.astype(np.float64) * ((x64 - x64[rows[0]]) ** 2).sum(1)
        p[rows[0]] = 0.0
        exp2 += p / p.sum()
    assert chi2(first, n * w / w.sum()) < 37.7
    assert chi2(second, exp2) < 37.7


@pytest.mark.parametrize("nc", [12, 100, 1000])
def test_recovers_separated_blobs(nc):
    m = max(20000, 40 * nc)
    x, lab, centers = kmeans_ref.blobs(m, 32, nc, seed=nc, spread=0.01)
    c = host(init_scalable(dev(x), n_clusters=nc, oversampling_factor=2.0, seed=5))
    blob, _ = kmeans_ref.assign(c, centers)
    assert sorted(blob) == list(range(nc))                        # exactly one seed per blob


@pytest.mark.parametrize("nc", [20, 200])
def test_quality_against_greedy(nc):
    """Thresholds from the model (test_kmeans_scalable.py): per seed a seeding cost 0.48-0.65 of greedy's; a converged
    inertia 0.84-1.21 of the greedy-seeded fit's for one seed, 0.93-1.01 on average over six.  Here: 0.75 per seed and
    1.1 for the sum over four seeds."""
    x, _, _ = kmeans_ref.blobs(100000, 32, nc, seed=nc + 1, spread=0.3)
    xd = dev(x)
    fa = fb = 0.0
    for seed in range(4):
        a = init_scalable(xd, n_clusters=nc, oversampling_factor=2.0, seed=seed)
        b = init_plus_plus(xd, n_clusters=nc, seed=seed)
        assert cluster_cost(xd, a) < 0.75 * cluster_cost(xd, b)
        fa += fit(KMeansParams(n_clusters=nc, seed=seed, oversampling_factor=2.0), xd).inertia
        fb += fit(KMeansParams(n_clusters=nc, seed=seed), xd).inertia
    assert fa < 1.1 * fb


def test_init_scalable_rejects_bad_factor():
    x = torch.zeros((10, 4), dtype=torch.float32, device="cuda")
    for bad in (0.0, -2.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            init_scalable(x, n_clusters=3, oversampling_factor=bad)


def test_fit_n_init_is_best_of_single_runs():
    x, _, _ = kmeans_ref.blobs(20000, 16, 8, seed=9, spread=0.4)
    xd = dev(x)
    runs = [fit(KMeansParams(n_clusters=8, max_iter=20, seed=10 + s, oversampling_factor=2.0), xd) for s in range(3)]
    best = min(range(3), key=lambda s: (runs[s].inertia, s))
    out = fit(KMeansParams(n_clusters=8, max_iter=20, seed=10, n_init=3, oversampling_factor=2.0), xd)
    assert host(out.centroids).tobytes() == host(runs[best].centroids).tobytes()
    assert out.inertia == runs[best].inertia and out.n_iter == runs[best].n_iter


def test_fit_graph_capture_equals_eager():
    x, _, _ = kmeans_ref.blobs(100000, 128, 64, seed=21, spread=0.5)
    xd = dev(x)
    p = KMeansParams(n_clusters=64, max_iter=15, tol=0.0, seed=2, oversampling_factor=2.0)
    a, b = fit(p, xd), fit(p, xd)
    assert host(a.centroids).tobytes() == host(b.centroids).tobytes()
    assert a.inertia == b.inertia and a.n_iter == b.n_iter == 15
    L = _lib.lib()
    m, k, nc = x.shape[0], x.shape[1], 64
    c = torch.empty((nc, k), dtype=torch.float32, device="cuda")
    inertia = torch.empty(1, dtype=torch.float64, device="cuda")
    n_iter = torch.empty(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(L.b2d_kmeans_scalable_workspace_bytes(m, k, nc, 2.0), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_kmeans_fit_scalable(ctypes.c_void_p(s.cuda_stream), nc, 15, 0.0, 2.0, 1, 2, 0, xd.data_ptr(), k,
                                             None, m, k, c.data_ptr(), inertia.data_ptr(), n_iter.data_ptr(),
                                             ws.data_ptr(), ws.numel()))
    c.zero_()
    ws.fill_(0xFF)
    g.replay()
    torch.cuda.synchronize()
    assert c.cpu().numpy().tobytes() == host(a.centroids).tobytes()
    assert inertia.item() == a.inertia and n_iter.item() == 15


def test_fit_weights():
    x, _, _ = kmeans_ref.blobs(20000, 16, 10, seed=4, spread=0.3)
    xd = dev(x)
    rng = np.random.default_rng(4)
    w = rng.uniform(0.0, 2.0, len(x)).astype(np.float32)
    w[:5000] = 0.0
    p = KMeansParams(n_clusters=10, seed=1, oversampling_factor=2.0)
    a = fit(p, xd, sample_weights=dev(w))
    b = fit(p, xd, sample_weights=dev(w))
    assert host(a.centroids).tobytes() == host(b.centroids).tobytes() and a.inertia == b.inertia
    assert np.isfinite(host(a.centroids)).all() and np.isfinite(a.inertia)
    wn = kmeans_ref.normalize(w, len(x)).astype(np.float64)
    _, d = kmeans_ref.assign(x, host(a.centroids))
    assert abs(a.inertia - (wn * d).sum()) <= 1e-4 * a.inertia
    w[7] = -1.0
    n = fit(p, xd, sample_weights=dev(w))
    assert np.isnan(n.inertia) and np.isfinite(host(n.centroids)).all()


def test_fit_without_factor_is_greedy():
    x, _, _ = kmeans_ref.blobs(20000, 16, 10, seed=6, spread=0.3)
    xd = dev(x)
    g = fit(KMeansParams(n_clusters=10, seed=3), xd)
    for f in (None, 0, 0.0):
        o = fit(KMeansParams(n_clusters=10, seed=3, oversampling_factor=f), xd)
        assert host(o.centroids).tobytes() == host(g.centroids).tobytes() and o.inertia == g.inertia
        assert o.n_iter == g.n_iter
    r = fit(KMeansParams(n_clusters=10, seed=3, init_method="Random"), xd)
    o = fit(KMeansParams(n_clusters=10, seed=3, init_method="Random", oversampling_factor=2.0), xd)
    assert host(o.centroids).tobytes() == host(r.centroids).tobytes()


@pytest.mark.parametrize("case", ["nc1", "nc_eq_m", "L_clamped", "few_distinct", "k1", "k320", "k784"])
def test_edges(case):
    rng = np.random.default_rng(11)
    m, k, nc, f = 3000, 16, 8, 2.0
    if case == "nc1":
        nc = 1
    elif case == "nc_eq_m":
        m, nc = 50, 50
    elif case == "L_clamped":
        m, nc, f = 30, 10, 5.0
    elif case.startswith("k"):
        k = int(case[1:])
    x = rng.normal(size=(m, k)).astype(np.float32)
    if case == "few_distinct":
        x = np.repeat(x[:5], m // 5, axis=0)
        nc = 10
    c, rows, wts = candidates(x, nc, f, seed=2)
    assert c.shape == (nc, k) and np.isfinite(c).all()
    assert len(rows) == ref.sizes(m, nc, f)[1] and rows.min() >= 0 and rows.max() < m
    assert wts.astype(np.float64).sum() == m
    if case in ("nc_eq_m", "L_clamped"):
        assert set(rows) == set(range(m))                       # every row once it has mass, then the massless rows
    o = fit(KMeansParams(n_clusters=nc, seed=2, oversampling_factor=f), dev(x))
    assert np.isfinite(host(o.centroids)).all() and np.isfinite(o.inertia)
