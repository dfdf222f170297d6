"""HDBSCAN's approximate_predict on the GPU, bit for bit against the oracle (tests/hdbscan_predict_ref.py): the
neighbours and their weights on their own (so that a walk error cannot hide behind the tree lookup), then labels and
probabilities for m from 1 to 2 10^4, both d, both metrics and min_samples in {1, 2, 5, 64}; both selection methods,
allow_single_cluster and cluster_selection_epsilon; queries that are fitted rows, in-blob points, far points, lattice
points with tied w and tied s, duplicate fitted rows and non-finite queries.  Then the identity property at 10^5 rows,
hdbscan_model's output against hdbscan's, independence from n_landmarks, the seed, the query order and the batching, a
pitched query array and a CUDA-graph replay."""
import functools

import numpy as np
import pytest

import hdbscan_predict_ref as R
import hdbscan_ref as H
from test_single_linkage_rbc_gpu import cuda, points

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

METRICS = ["sqeuclidean", "euclidean"]


def queries(x, n, seed):
    """fitted rows, points near them, uniform points over the data's box and beyond, and lattice points (half-integer
    and integer: tied s and tied w on lattice data)"""
    r = np.random.default_rng(seed)
    m, d = x.shape
    lo, hi = x.min(0), x.max(0)
    span = np.maximum(hi - lo, 1e-30)
    parts = [x[r.integers(0, m, n)],
             x[r.integers(0, m, n)] + (r.normal(0, 0.02, (n, d)) * span).astype(np.float32),
             (lo + r.random((n, d)) * span).astype(np.float32),
             (lo - span + 3 * r.random((n // 4 + 1, d)) * span).astype(np.float32),
             (np.round(lo + r.random((n // 4 + 1, d)) * span) + r.integers(0, 2, (n // 4 + 1, 1)) * 0.5).astype(np.float32)]
    return np.concatenate(parts).astype(np.float32)


@functools.lru_cache(maxsize=None)
def ref_tree(m, d, seed, kind, ms):
    """the oracle's tree in the s domain (cached across metrics and selections)"""
    x = points(m, d, seed, kind)
    return x, H.mr_tree(x, ms)


def model_ref(m, d, seed, kind, mcs, ms, metric, method="eom", single=False, eps=0.0):
    x, tree = ref_tree(m, d, seed, kind, ms)
    return x, R.fit(x, mcs, ms, method, single, eps, metric, tree)


def fit_gpu(x, mcs, ms, metric, method="eom", single=False, eps=0.0, **kw):
    from raft_b200.cluster import hdbscan_model
    return hdbscan_model(x if torch.is_tensor(x) else cuda(x), min_cluster_size=mcs, min_samples=ms,
                         cluster_selection_epsilon=eps, cluster_selection_method=method, allow_single_cluster=single,
                         metric=metric, **kw)


def predict_gpu(model, q):
    from raft_b200.cluster import approximate_predict
    p = approximate_predict(model, q if torch.is_tensor(q) else cuda(q))
    return tuple(t.cpu().numpy() for t in p)


def same(got, want, what=""):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32)) if got.itemsize == 4 else \
        np.flatnonzero(got != want)
    assert not len(bad), (what, bad[:8], got[bad[:8]], want[bad[:8]])


def check(m, d, seed, kind, mcs, ms, metric, method="eom", single=False, eps=0.0, nq=200, extra=None):
    x, ref = model_ref(m, d, seed, kind, mcs, ms, metric, method, single, eps)
    q = queries(x, nq, seed + 1)
    if extra is not None:
        q = np.concatenate([q, extra]).astype(np.float32)
    want = R.predict(ref, q)
    got = predict_gpu(fit_gpu(x, mcs, ms, metric, method, single, eps), q)
    same(got[2], want[2], "neighbors")   # the walk first
    same(got[3], want[3], "weights")
    same(got[0], want[0], "labels")
    same(got[1], want[1], "probabilities")
    return got


NON_FINITE = np.array([[np.nan, 0, 0], [0, np.inf, 0], [-np.inf, 1, 1], [np.nan, np.nan, np.nan]], np.float32)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("ms", [1, 2, 5, 64])
@pytest.mark.parametrize("m", [1, 2, 3, 70, 1000, 5000])
def test_shapes(m, d, ms, metric):
    if ms > m:
        pytest.skip("min_samples > m")
    got = check(m, d, 10 * m + d, "uniform", 5, ms, metric, extra=NON_FINITE[:, :d])
    assert (got[0][-4:] == -1).all() and (got[2][-4:] == -1).all()


@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("ms", [5, 64])
def test_twenty_thousand(d, ms):
    for metric in METRICS:
        check(20000, d, 7 + d, "blobs", 50, ms, metric, nq=300)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("kind", ["lattice", "duplicates", "ring", "cancellation", "subnormal", "dense_ball", "blobs"])
def test_adversarial(kind, d, metric):
    for ms in (1, 5, 64):
        check(3000, d, 3, kind, 10, ms, metric)


@pytest.mark.parametrize("method", ["eom", "leaf"])
@pytest.mark.parametrize("single", [False, True])
@pytest.mark.parametrize("eps", [0.0, 0.05, 5.0])
def test_selection(method, single, eps):
    for kind, mcs, ms in (("blobs", 15, 5), ("uniform", 5, 3), ("duplicates", 20, 20), ("uniform", 400, 10)):
        check(2000, 2, 5, kind, mcs, ms, "euclidean", method, single, eps)


def test_far_points_are_noise_and_blob_centres_take_their_blob():
    from test_hdbscan_predict import two_blobs
    lab, prob, nn, w = predict_gpu(fit_gpu(two_blobs(), 20, 5, "euclidean"),
                                   np.array([[-10, 0], [10, 0], [0, 1e4]], np.float32))
    assert lab.tolist() == [0, 1, -1] and prob.tolist() == [1.0, 1.0, 0.0]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
def test_identity_property_at_1e5(d, metric):
    """a fitted row given back (no duplicate rows) gets the fit's label and probability, and itself as neighbour"""
    x = points(100000, d, 31 + d, "blobs")
    assert len(np.unique(x, axis=0)) == len(x)
    model = fit_gpu(x, 50, 10, metric)
    lab, prob, nn, w = predict_gpu(model, x)
    same(nn, np.arange(len(x), dtype=np.int32), "neighbors")
    same(lab, model.output.labels.cpu().numpy(), "labels")
    same(prob, model.output.probabilities.cpu().numpy(), "probabilities")
    assert model.output.n_clusters >= 2


def test_model_output_is_hdbscans():
    from raft_b200.cluster import hdbscan
    x = cuda(points(6000, 3, 21, "blobs"))
    for kw in (dict(), dict(cluster_selection_method="leaf", allow_single_cluster=True, cluster_selection_epsilon=0.5),
               dict(metric="sqeuclidean", min_samples=64)):
        a = hdbscan(x, min_cluster_size=20, **kw)
        b = fit_gpu(x, 20, kw.pop("min_samples", None), kw.pop("metric", "euclidean"),
                    kw.get("cluster_selection_method", "eom"), kw.get("allow_single_cluster", False),
                    kw.get("cluster_selection_epsilon", 0.0)).output
        for g, w in ((b.labels, a.labels), (b.probabilities, a.probabilities)) + tuple(zip(b.mst, a.mst)):
            same(g.cpu().numpy(), w.cpu().numpy())
        assert b.n_clusters == a.n_clusters


def test_independent_of_landmarks_seed_order_and_batching():
    x = points(6000, 2, 22, "blobs")
    q = queries(x, 2000, 23)
    want = predict_gpu(fit_gpu(x, 20, 8, "euclidean"), q)
    for kw in (dict(n_landmarks=1), dict(n_landmarks=6000), dict(n_landmarks=17, seed=5), dict(seed=123)):
        got = predict_gpu(fit_gpu(x, 20, 8, "euclidean", **kw), q)
        for g, w in zip(got, want):
            same(g, w)
    model = fit_gpu(x, 20, 8, "euclidean")
    perm = np.random.default_rng(1).permutation(len(q))
    got = predict_gpu(model, q[perm])
    for g, w in zip(got, want):
        same(g, w[perm])
    parts = [predict_gpu(model, q[a:b]) for a, b in ((0, 1), (1, 777), (777, len(q)))]
    for k in range(4):
        same(np.concatenate([p[k] for p in parts]), want[k])
    assert all(len(t) == 0 for t in predict_gpu(model, np.zeros((0, 2), np.float32)))


def test_pitched_queries_and_cuda_graph_replay():
    x = points(5000, 3, 24, "blobs")
    q = queries(x, 1000, 25)
    model = fit_gpu(x, 25, 7, "sqeuclidean")
    want = predict_gpu(model, q)
    qp = torch.zeros((len(q), 7), dtype=torch.float32, device="cuda")
    qp[:, :3] = cuda(q)
    for g, w in zip(predict_gpu(model, qp[:, :3]), want):
        same(g, w)
    # the C call captured on a side stream, then replayed on new query values
    import ctypes
    from raft_b200 import _lib
    L = _lib.lib()
    qd = cuda(q[::-1].copy())
    out = [torch.full((len(q),), -7, dtype=dt, device="cuda") for dt in (torch.int32, torch.float32, torch.int32,
                                                                          torch.float32)]
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_hdbscan_rbc_approximate_predict(
            ctypes.c_void_p(s.cuda_stream), model.buffer.data_ptr(), model.m, model.d, model.metric, model.n_landmarks,
            model.min_samples, qd.data_ptr(), 3, len(q), *[t.data_ptr() for t in out]))
    qd.copy_(cuda(q))
    for _ in range(2):
        for t in out:
            t.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        for t, w in zip(out, want):
            same(t.cpu().numpy(), w)
