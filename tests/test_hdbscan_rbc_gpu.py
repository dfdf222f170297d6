"""HDBSCAN on the random ball cover on the GPU: the mutual-reachability tree equals the oracle's (tests/hdbscan_ref.py:
Prim's algorithm under the contract's strict edge order on the fp32 term-by-term pair values) byte for byte, and the
labels, probabilities and cluster count equal the oracle's tree stages on it exactly.  Covered: m from 1 to 2 10^4, both d,
both metrics and min_samples in {1, 2, 5, 64}; the ball cover tests' hard data (an integer lattice with massive ties,
exact duplicates, rows on a ball's radius, a 1e4 offset with a 1e-2 spread, 1e-20 coordinates, a dense ball with far
outliers, blobs); both selection methods, allow_single_cluster and cluster_selection_epsilon; min_samples = 1 against
cluster.emst; independence from n_landmarks, the seed and repeated calls; a non-finite X."""
import functools

import numpy as np
import pytest

import hdbscan_ref as H
from test_single_linkage_rbc_gpu import cuda, points

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

METRICS = ["sqeuclidean", "euclidean"]


@functools.lru_cache(maxsize=None)
def ref_tree(m, d, seed, kind, ms):
    """the oracle's tree in the s domain (cached across metrics)"""
    x = points(m, d, seed, kind)
    src, dst, w, _ = H.mr_tree(x, ms)
    return x, src, dst, w


def ref(m, d, seed, kind, ms, metric, mcs, method="eom", single=False, eps=0.0):
    x, src, dst, w = ref_tree(m, d, seed, kind, ms)
    if metric == "euclidean":
        w = np.sqrt(w, dtype=np.float32)
    lab, prob, n = H.tree_labels(src, dst, w, m, mcs, method, single, eps)
    return x, (src, dst, w), lab, prob.astype(np.float32), n


def run(x, metric, mcs, ms, method="eom", single=False, eps=0.0, **kw):
    from raft_b200.cluster import hdbscan
    o = hdbscan(x if torch.is_tensor(x) else cuda(x), min_cluster_size=mcs, min_samples=ms, cluster_selection_epsilon=eps,
                cluster_selection_method=method, allow_single_cluster=single, metric=metric, **kw)
    tree = tuple(t.cpu().numpy() for t in o.mst)
    return tree, o.labels.cpu().numpy(), o.probabilities.cpu().numpy(), o.n_clusters


def same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    assert got.tobytes() == want.tobytes(), (np.flatnonzero(got != want)[:8], got[:8], want[:8])


def check(m, d, seed, kind, ms, metric, mcs, method="eom", single=False, eps=0.0, **kw):
    x, tree, lab, prob, n = ref(m, d, seed, kind, ms, metric, mcs, method, single, eps)
    gtree, glab, gprob, gn = run(x, metric, mcs, ms, method, single, eps, **kw)
    for g, w in zip(gtree, tree):
        same(g, w)
    same(glab, lab)
    same(gprob, prob)
    assert gn == n


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("ms", [1, 2, 5, 64])
@pytest.mark.parametrize("m", [1, 2, 3, 70, 1000, 5000])
def test_shapes(m, d, ms, metric):
    if ms > m:
        pytest.skip("min_samples > m")
    check(m, d, 10 * m + d, "uniform", ms, metric, 5)


@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("ms", [5, 64])
def test_twenty_thousand(d, ms):
    for metric in METRICS:
        check(20000, d, 7 + d, "blobs", ms, metric, 50)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("kind", ["lattice", "duplicates", "ring", "cancellation", "subnormal", "dense_ball", "blobs"])
def test_adversarial(kind, d, metric):
    for ms in (1, 5, 64):
        check(3000, d, 3, kind, ms, metric, 10)


@pytest.mark.parametrize("method", ["eom", "leaf"])
@pytest.mark.parametrize("single", [False, True])
@pytest.mark.parametrize("eps", [0.0, 0.05, 5.0])
def test_selection(method, single, eps):
    for kind, mcs, ms in (("blobs", 15, 5), ("uniform", 5, 3), ("duplicates", 20, 20), ("uniform", 400, 10)):
        check(2000, 2, 5, kind, ms, "euclidean", mcs, method, single, eps)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
def test_min_samples_one_is_the_emst(d, metric):
    from raft_b200.cluster import emst
    x = cuda(points(4000, d, 11, "blobs"))
    e = emst(x, metric=metric)
    tree, *_ = run(x, metric, 5, 1)
    for g, w in zip(tree, e):
        same(g, w.cpu().numpy())


def test_independent_of_landmarks_seed_and_repeats():
    x = cuda(points(6000, 3, 21, "blobs"))
    want = run(x, "euclidean", 20, 8)
    for kw in (dict(n_landmarks=1), dict(n_landmarks=6000), dict(n_landmarks=17, seed=5), dict(seed=123), {}, {}):
        got = run(x, "euclidean", 20, 8, **kw)
        for g, w in zip(got[0], want[0]):
            same(g, w)
        same(got[1], want[1])
        same(got[2], want[2])
        assert got[3] == want[3]


def test_pitched_x():
    x = points(3000, 2, 4, "blobs")
    xp = np.zeros((3000, 5), np.float32)
    xp[:, :2] = x
    got = run(cuda(xp)[:, :2], "sqeuclidean", 10, 5)
    want = run(cuda(x), "sqeuclidean", 10, 5)
    for g, w in zip(got[0] + got[1:3], want[0] + want[1:3]):
        same(g, w)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_x_raises(bad):
    from raft_b200.cluster import hdbscan
    x = points(500, 3, 2)
    x[77, 1] = bad
    with pytest.raises(ValueError, match="non-finite"):
        hdbscan(cuda(x))
