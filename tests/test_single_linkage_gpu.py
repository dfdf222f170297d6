"""single_linkage and its minimum spanning forest on the GPU: b2d_mst against Kruskal edge for edge, single_linkage on
complete graphs against scipy, on blobs against the reference computed from the device's own kNN, connect_components on
separated blobs and on clusters of exact duplicates, determinism and edge cases."""
import numpy as np
import pytest

import single_linkage_ref as ref

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
hierarchy = pytest.importorskip("scipy.cluster.hierarchy")


def _sl(x, n_clusters, metric="euclidean", c=15):
    from raft_b200.cluster import single_linkage
    o = single_linkage(torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda(), n_clusters, metric=metric, c=c)
    return (o.children.cpu().numpy(), o.deltas.cpu().numpy(), o.sizes.cpu().numpy(), o.labels.cpu().numpy(),
            o.n_connected_components)


def _graph(rng, n, e, integer, pieces=1):
    """A random edge list: integer weights (many ties) or floats, duplicate and reversed edges, self-loops; with
    pieces > 1 the vertices split into that many ranges with no edge between them."""
    cut = np.linspace(0, n, pieces + 1).astype(int)
    part = rng.integers(0, pieces, e)
    lo, hi = cut[part], cut[part + 1]
    src = lo + (rng.random(e) * (hi - lo)).astype(int)
    dst = lo + (rng.random(e) * (hi - lo)).astype(int)
    w = rng.integers(0, 8, e).astype(np.float32) if integer else rng.standard_normal(e).astype(np.float32)
    k = e // 10   # duplicates and reversed copies of earlier edges, self-loops
    src[-k:], dst[-k:], w[-k:] = dst[:k], src[:k], w[:k]
    src[-2 * k:-k], dst[-2 * k:-k], w[-2 * k:-k] = src[:k], dst[:k], w[:k] + np.float32(rng.integers(0, 2))
    dst[-3 * k:-2 * k] = src[-3 * k:-2 * k]
    return src.astype(np.int32), dst.astype(np.int32), w


@pytest.mark.parametrize("n,e,integer,pieces", [(50, 200, True, 1), (1000, 3000, True, 3), (1000, 3000, False, 1),
                                                (5000, 9000, False, 7), (20000, 200000, True, 1), (3000, 2000, True, 1)])
def test_mst_equals_kruskal(n, e, integer, pieces):
    from raft_b200.cluster import mst
    rng = np.random.default_rng(n + e + pieces)
    src, dst, w = _graph(rng, n, e, integer, pieces)
    o = mst(torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(), torch.from_numpy(w).cuda(), n)
    chosen, colour = ref.kruskal(src, dst, w, n)
    assert (o.src.cpu().numpy() == src[chosen]).all()
    assert (o.dst.cpu().numpy() == dst[chosen]).all()
    assert o.weights.cpu().numpy().tobytes() == w[chosen].tobytes()
    assert (o.colour.cpu().numpy() == colour).all()
    assert len(chosen) == n - len(np.unique(colour))


def test_mst_empty_and_out_of_range_edges():
    from raft_b200.cluster import mst
    src = torch.tensor([0, 5, -1, 1], dtype=torch.int32, device="cuda")
    dst = torch.tensor([1, 0, 2, 2], dtype=torch.int32, device="cuda")
    w = torch.tensor([3.0, 1.0, 0.0, 2.0], device="cuda")
    o = mst(src, dst, w, 4)
    assert o.src.tolist() == [1, 0] and o.dst.tolist() == [2, 1] and o.colour.tolist() == [0, 0, 0, 3]
    e = torch.empty(0, dtype=torch.int32, device="cuda")
    o = mst(e, e, torch.empty(0, device="cuda"), 3)
    assert len(o.src) == 0 and o.colour.tolist() == [0, 1, 2]


def _scipy(x, n_clusters):
    Z = hierarchy.linkage(x.astype(np.float64), method="single", metric="euclidean")
    lab = hierarchy.fcluster(Z, n_clusters, criterion="maxclust")
    return Z, ref.canonical_labels(lab)


@pytest.mark.parametrize("m,d", [(5, 3), (33, 8), (64, 40), (64, 300)])
def test_complete_graph_equals_scipy(m, d):
    x = np.random.default_rng(m * d).standard_normal((m, d)).astype(np.float32)
    for nc in (1, 2, 3, m // 2, m):
        ch, de, sz, lab, ncomp = _sl(x, nc, c=64)
        Z, slab = _scipy(x, nc)
        assert ncomp == 1
        assert (ch == Z[:, :2].astype(np.int64)).all() and (sz == Z[:, 3].astype(np.int64)).all()
        np.testing.assert_allclose(de, Z[:, 2], rtol=1e-5)
        assert (lab == slab).all(), nc


def _blobs(m, d, n_blobs, spread, seed, sep=10.0):
    rng = np.random.default_rng(seed)
    centers = rng.uniform(-sep, sep, (n_blobs, d))
    y = rng.integers(0, n_blobs, m)
    return (centers[y] + spread * rng.standard_normal((m, d))).astype(np.float32), y


@pytest.mark.parametrize("m,d,metric", [(2000, 16, "euclidean"), (7000, 5, "sqeuclidean"), (20000, 32, "euclidean")])
def test_same_algorithm_as_reference(m, d, metric):
    from raft_b200.neighbors import brute_force
    x, _ = _blobs(m, d, 4, 3.0, seed=m, sep=1.0)   # overlapping blobs: a connected kNN graph
    nb = ref.n_neighbors(m)
    dist, idx = brute_force.knn(torch.from_numpy(x).cuda(), torch.from_numpy(x).cuda(), nb, metric="sqeuclidean")
    dist, idx = dist.cpu().numpy(), idx.cpu().numpy()
    sq = metric == "euclidean"
    for nc in (1, 4, 50):
        ch, de, sz, lab, ncomp = _sl(x, nc, metric=metric)
        assert ncomp == 1   # (connect_components is checked against scipy by the tests below)
        rch, rde, rsz, rlab, rncomp = ref.single_linkage_from_knn(x, idx, dist, nc, sqrt=sq)
        assert rncomp == 1
        assert (ch == rch).all() and (sz == rsz).all() and (lab == rlab).all()
        assert de.tobytes() == rde.astype(np.float32).tobytes()


@pytest.mark.parametrize("metric", ["euclidean", "sqeuclidean"])
def test_connect_components_separated_blobs(metric):
    n_blobs, m, d = 6, 3000, 8
    x, y = _blobs(m, d, n_blobs, 1.0, seed=5, sep=100.0)
    ch, de, sz, lab, ncomp = _sl(x, n_blobs, metric=metric)
    assert ncomp >= n_blobs
    assert sz[-1] == m and len(np.unique(ch)) == 2 * (m - 1) and ch.max() == 2 * m - 3
    Z, _ = _scipy(x, n_blobs)
    want = Z[-(n_blobs - 1):, 2] if metric == "euclidean" else Z[-(n_blobs - 1):, 2] ** 2
    np.testing.assert_allclose(np.sort(de)[-(n_blobs - 1):], want, rtol=1e-4)
    assert (lab == ref.canonical_labels(y)).all()


def test_fragmented_duplicates_use_row_chunks():
    # 500 clusters of 40 identical rows each (n_nb = 29): 500 components, so the connect step's adjacency is cut into
    # row chunks (128 m / c = 5120 rows)
    rng = np.random.default_rng(11)
    k, rep, d = 500, 40, 8
    centers = rng.uniform(-50, 50, (k, d)).astype(np.float32)
    y = rng.permutation(np.repeat(np.arange(k), rep))
    x = centers[y]
    ch, de, sz, lab, ncomp = _sl(x, k, metric="sqeuclidean")
    assert ncomp == k
    assert sz[-1] == k * rep
    assert de[:k * rep - k].max() <= 1e-3 * de[k * rep - k:].min()   # copies merge first (at the kNN's ~0)
    Z = hierarchy.linkage(centers.astype(np.float64), method="single")
    np.testing.assert_allclose(de[-(k - 1):], Z[:, 2] ** 2, rtol=1e-3)
    assert (lab == ref.canonical_labels(y)).all()


def test_deterministic():
    x, _ = _blobs(12000, 24, 9, 1.5, seed=2, sep=30.0)
    a, b = _sl(x, 9), _sl(x, 9)
    for u, v in zip(a[:4], b[:4]):
        assert u.tobytes() == v.tobytes()
    assert a[4] == b[4]


def test_edge_cases():
    x1 = np.ones((1, 4), np.float32)
    ch, de, sz, lab, ncomp = _sl(x1, 1)
    assert ch.shape == (0, 2) and len(de) == 0 and lab.tolist() == [0] and ncomp == 1
    x2 = np.array([[0, 0], [3, 4]], np.float32)
    ch, de, sz, lab, ncomp = _sl(x2, 1)
    assert ch.tolist() == [[0, 1]] and de.tolist() == [5.0] and sz.tolist() == [2] and lab.tolist() == [0, 0]
    assert _sl(x2, 2)[3].tolist() == [0, 1]
    x = np.random.default_rng(3).standard_normal((300, 6)).astype(np.float32)
    assert (_sl(x, 300)[3] == np.arange(300)).all()
    assert (_sl(x, 1)[3] == 0).all()


def test_errors():
    from raft_b200 import LogicError
    x = np.random.default_rng(0).standard_normal((100, 4)).astype(np.float32)
    x[17, 2] = np.nan
    with pytest.raises(LogicError, match="non-finite"):
        _sl(x, 3)
    x[17, 2] = np.inf
    with pytest.raises(LogicError, match="non-finite"):
        _sl(x, 3)
    with pytest.raises(LogicError, match="lower c"):
        _sl(np.zeros((1000, 4), np.float32), 3, c=60)
    with pytest.raises(LogicError):
        _sl(np.zeros((10, 4), np.float32), 11)
    with pytest.raises(LogicError):
        _sl(np.zeros((10, 4), np.float32), 2, metric="cosine")
