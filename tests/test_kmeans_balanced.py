"""Balanced k-means without a GPU: the fine allocation of the model (tests/kmeans_balanced_ref.py), the model's balance
and quality against plain Lloyd, the ABI declarations, every argument error of b2d_kmeans_balanced_fit, its workspace
query and the recorded workspace contract (tests/golden/kmeans_balanced_workspace_contract.json), and the Python
parameters."""
import os
import re

import numpy as np
import pytest

import kmeans_balanced_ref as ref
import kmeans_ref
from raft_b200 import _lib
from test_workspace_contract import load, replay_bytes, replay_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_WORKSPACE
NEW = ["b2d_kmeans_balanced_workspace_bytes", "b2d_kmeans_balanced_fit"]
CONTRACT = "kmeans_balanced_workspace_contract.json"


def fit(nc=4, n_iters=20, x=P, ldx=8, m=100, k=8, c=P, labels=None, sizes=None, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_kmeans_balanced_fit(None, nc, n_iters, 0, x, ldx, m, k, c, labels, sizes, ws, wsb)


def status(rc):
    return rc, _lib.lib().b2d_last_error().decode()


def check_alloc(S, nc):
    a = ref.allocate(S, nc)
    assert sum(a) == nc, (S, nc, a)
    for s, n in zip(S, a):
        assert n >= 0
        if s > 0:
            assert n >= 1, (S, nc, a)
        if sum(S) >= nc:
            assert n <= s, (S, nc, a)
    return a


def test_groups():
    assert [ref.groups(n) for n in (1, 2, 3, 4, 6, 7, 1024, 16384, 65536)] == [1, 1, 2, 2, 2, 3, 32, 128, 256]


def test_allocation_edges():
    assert check_alloc([10], 7) == [7]                      # G = 1
    assert check_alloc([5, 0, 5], 4) == [2, 0, 2]           # an empty mesocluster gets nothing
    assert check_alloc([3, 3, 3], 9) == [3, 3, 3]           # n_clusters = m: one row per cluster
    assert check_alloc([1, 1, 7], 9) == [1, 1, 7]
    assert check_alloc([1, 2, 1], 3) == [1, 1, 1]           # remainders 3, 2, 3 of 4: ties to the lower g
    assert check_alloc([1, 1, 98], 10) == [1, 1, 8]         # the minimum of one comes from the largest a / S
    assert check_alloc([0, 0], 3) == [3, 0]                 # no finite row: everything to mesocluster 0


def test_allocation_random():
    rng = np.random.default_rng(0)
    for _ in range(500):
        G = int(rng.integers(1, 40))
        S = rng.integers(0, 50, size=G) * (rng.random(G) < 0.8)
        if S.sum() == 0:
            S[0] = 1
        nc = int(rng.integers(max(G, 1), max(G, S.sum()) + 1))   # G <= n_clusters, as G = round(sqrt(n_clusters))
        check_alloc(list(S), nc)


def spreads(sizes):
    avg = sizes.sum() / len(sizes)
    return sizes.min() / avg, sizes.max() / avg


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_model_balance_and_quality(seed):
    """On uniform data and on a skewed mixture (4000 x 8, 64 clusters, 10 iterations; 90 % of the rows in one tight
    blob) the model's cluster sizes stay within [0.25, 1.7] of the average (measured over seeds 0-2: 0.34-0.70 /
    1.31-1.49).  Its inertia is within 1.3 of Lloyd's from the same
    strided rows (measured: 1.01-1.16; balance costs some inertia on the skewed data)."""
    for x in (uniform(seed), skewed(seed)):
        c, lab, sizes = ref.fit(x, 64, 10, seed)
        assert (sizes == np.bincount(lab, minlength=64)).all()
        lo, hi = spreads(sizes)
        assert lo >= 0.25 and hi <= 1.7, (lo, hi)
        _, _, inertia, _ = kmeans_ref.lloyd(x, x[(np.arange(64) * len(x)) // 64], 20, 0.0)
        assert kmeans_ref.cost(x, c) < 1.3 * inertia


def uniform(seed, m=4000, k=8):
    return np.random.default_rng(seed).uniform(-1, 1, size=(m, k)).astype(np.float32)


def skewed(seed, m=4000, k=8):
    """90 % of the rows in one tight blob, the rest in a wide one."""
    rng = np.random.default_rng(seed + 100)
    big = rng.normal(0, 0.05, size=(m - m // 10, k))
    rest = rng.normal(0, 1.0, size=(m // 10, k)) + 4
    return np.concatenate([big, rest]).astype(np.float32)[rng.permutation(m)]


def test_model_nan_rows_and_stages():
    x, _, _ = kmeans_ref.blobs(600, 4, 6, seed=5, spread=0.02)
    x[[3, 77, 500]] = np.nan
    x[10, 2] = np.inf
    c, lab, sizes, st = ref.fit(x, 20, 5, 0, stages=True)
    assert (lab[[3, 10, 77, 500]] == -1).all() and (lab >= 0).sum() == 596
    assert np.isfinite(c).all() and sizes.sum() == 596
    assert sum(st["alloc"]) == 20 and len(st["alloc"]) == ref.groups(20)
    # the fine stage never assigns across mesoclusters
    F = np.concatenate([[0], np.cumsum(st["alloc"])])
    ok = st["meso"] >= 0
    assert ((st["fine_labels"][ok] >= F[st["meso"][ok]]) & (st["fine_labels"][ok] < F[st["meso"][ok] + 1])).all()


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(_lib.lib(), s)


def test_argument_errors():
    assert status(fit(nc=0)) == (E, "n_clusters must be in [1, m]")
    assert status(fit(nc=101)) == (E, "n_clusters must be in [1, m]")
    assert status(fit(x=None)) == (E, "null x / centroids")
    assert status(fit(c=None)) == (E, "null x / centroids")
    assert status(fit(ldx=7)) == (E, "leading dimension smaller than k")
    assert status(fit(k=0)) == (E, "k must be in [1, 2^24]")
    assert status(fit(k=-1)) == (E, "negative extent")
    assert status(fit(m=2 ** 31)) == (E, "m must be below 2^31")
    for n in (0, -1):
        assert status(fit(n_iters=n)) == (E, "n_iters must be >= 1")
    need = _lib.lib().b2d_kmeans_balanced_workspace_bytes(100, 8, 4)
    assert fit(ws=None, wsb=need) == W
    assert fit(wsb=need - 1) == W
    assert fit(ws=P * 256 + 8, wsb=need) == E   # not 256-byte aligned
    assert fit(m=0, nc=0, x=None, c=None, n_iters=0) == _lib.B2D_OK


def test_workspace_query():
    L = _lib.lib()
    wb = L.b2d_kmeans_balanced_workspace_bytes
    for args in ((-1, 8, 2), (10, -1, 2), (10, 8, -1)):
        assert wb(*args) == SIZE_MAX
    for m, k, nc in ((1, 1, 1), (100, 8, 4), (5000, 96, 40), (10 ** 6, 128, 1024), (10 ** 6, 128, 65536)):
        b = wb(m, k, nc)
        # at least x sorted by mesocluster and one k-means workspace for n_clusters
        assert b % 1024 == 0 and b >= 4 * m * k + L.b2d_kmeans_workspace_bytes(m, k, nc), (m, k, nc)
    assert wb(10 ** 6, 128, 1024) < wb(10 ** 6, 128, 65536)


def test_workspace_contract_bytes():
    rows = replay_bytes(load(CONTRACT), "b2d_kmeans_balanced_workspace_bytes")
    for m, k, nc, want in rows:
        assert (want == SIZE_MAX) == (min(m, k, nc) < 0), (m, k, nc)


def test_workspace_contract_errors():
    assert replay_errors(load(CONTRACT)) == 6


def test_python_params_and_exports():
    import raft_b200
    import raft_b200.cluster as cl
    from raft_b200.cluster.kmeans_balanced import KMeansBalancedParams
    p = KMeansBalancedParams()
    assert (p.n_iters, p.metric, p.seed) == (20, "sqeuclidean", 0)
    for bad in ("cosine", "inner_product", "L1"):
        with pytest.raises(_lib.LogicError):
            KMeansBalancedParams(metric=bad)
    with pytest.raises(ValueError):
        KMeansBalancedParams(n_iters=0)
    assert cl.fit is cl.kmeans.fit and cl.kmeans_balanced.fit is not cl.fit
    assert not hasattr(raft_b200, "KMeansBalancedParams") and not hasattr(cl, "fit_predict")
