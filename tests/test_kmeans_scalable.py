"""k-means|| without a GPU: the ABI declarations, the argument checks and workspace query of b2d_kmeans_init_scalable /
b2d_kmeans_fit_scalable, their recorded workspace contract (tests/golden/kmeans_scalable_workspace_contract.json), the
routing rules of KMeansParams.oversampling_factor, and the numpy model (tests/kmeans_scalable_ref.py) against greedy
k-means++."""
import os
import re

import numpy as np
import pytest

import kmeans_ref
import kmeans_scalable_ref as ref
from raft_b200 import _lib
from test_workspace_contract import load, replay_bytes, replay_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE
NEW = ["b2d_kmeans_scalable_workspace_bytes", "b2d_kmeans_init_scalable", "b2d_kmeans_fit_scalable"]
CONTRACT = "kmeans_scalable_workspace_contract.json"


def init(x=P, ldx=8, w=None, m=100, k=8, nc=4, f=2.0, c=P, cand=None, cw=None, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_kmeans_init_scalable(None, x, ldx, w, m, k, nc, f, 0, c, cand, cw, ws, wsb)


def fit(nc=4, max_iter=10, tol=1e-4, f=2.0, n_init=1, x=P, ldx=8, w=None, m=100, k=8, c=P, inertia=P, n_iter=P,
        ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_kmeans_fit_scalable(None, nc, max_iter, tol, f, n_init, 0, 0, x, ldx, w, m, k, c, inertia,
                                              n_iter, ws, wsb)


def status(rc):
    return rc, _lib.lib().b2d_last_error().decode()


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(_lib.lib(), s)


@pytest.mark.parametrize("call", [init, fit])
def test_argument_errors(call):
    for f in (0.0, -1.0, float("nan"), float("inf")):
        assert status(call(f=f)) == (E, "oversampling_factor must be finite and > 0"), f
    assert status(call(nc=0)) == (E, "n_clusters must be in [1, m]")
    assert status(call(nc=101)) == (E, "n_clusters must be in [1, m]")
    assert status(call(x=None)) == (E, "null x / centroids")
    assert status(call(c=None)) == (E, "null x / centroids")
    assert status(call(ldx=7)) == (E, "leading dimension smaller than k")
    assert status(call(k=0)) == (E, "k must be in [1, 2^24]")
    assert status(call(m=2 ** 31)) == (E, "m must be below 2^31")
    # L = 2^29 rows per round: C = 1 + 2^32 candidates
    assert status(call(m=2 ** 30, nc=2 ** 28, f=2.0)) == \
        (U, "k-means|| candidate set of 1 + 8 L rows must stay below 2^31")
    need = _lib.lib().b2d_kmeans_scalable_workspace_bytes(100, 8, 4, 2.0)
    assert call(ws=None, wsb=need) == W
    assert call(wsb=need - 1) == W
    assert call(ws=P * 256 + 8, wsb=need) == E   # not 256-byte aligned
    assert call(m=0, nc=0, x=None, c=None, f=float("nan")) == _lib.B2D_OK


def test_fit_argument_errors():
    assert status(fit(inertia=None)) == (E, "null inertia / n_iter")
    assert status(fit(n_iter=None)) == (E, "null inertia / n_iter")
    assert status(fit(max_iter=-1)) == (E, "max_iter must be >= 0")
    assert status(fit(tol=float("nan"))) == (E, "tol must be >= 0")
    assert status(fit(n_init=0)) == (E, "n_init must be >= 1")


def test_workspace_query():
    L = _lib.lib()
    wb = L.b2d_kmeans_scalable_workspace_bytes
    for args in ((-1, 8, 2), (10, -1, 2), (10, 8, -1)):
        assert wb(*args, 2.0) == SIZE_MAX
    for f in (0.0, -0.5, float("nan"), float("inf")):
        assert wb(100, 8, 4, f) == SIZE_MAX
    assert wb(2 ** 30, 8, 2 ** 28, 2.0) == SIZE_MAX
    for m, k, nc in ((1, 1, 1), (100, 8, 4), (5000, 96, 40), (10 ** 6, 128, 1024), (10 ** 6, 128, 10 ** 5)):
        for f in (0.01, 0.5, 2.0, 1e6):
            b = wb(m, k, nc, f)
            assert b % 1024 == 0 and b >= L.b2d_kmeans_workspace_bytes(m, k, nc), (m, k, nc, f)
    assert wb(10 ** 6, 128, 1024, 2.0) < wb(10 ** 6, 128, 1024, 4.0)


def test_workspace_contract_bytes():
    rows = replay_bytes(load(CONTRACT), "b2d_kmeans_scalable_workspace_bytes")
    for m, k, nc, f, want in rows:
        bad = min(m, k, nc) < 0 or not (0 < f < float("inf")) or (nc >= 0 and m >= 0 and ref.sizes(m, nc, f)[1] >= 2 ** 31)
        assert (want == SIZE_MAX) == bad, (m, k, nc, f)


def test_workspace_contract_errors():
    assert replay_errors(load(CONTRACT)) == 9


def test_sizes():
    assert ref.sizes(10 ** 6, 1024, 2.0) == (2048, 16385)
    assert ref.sizes(10 ** 6, 1000, 0.01) == (125, 1001)     # the (n_clusters - 1) / 8 floor: C >= n_clusters
    assert ref.sizes(5, 5, 2.0) == (5, 41)                   # L clamped to m
    for m, nc, f in ((1, 1, 0.1), (100, 100, 0.001), (37, 20, 3.0), (10 ** 6, 4096, 0.5)):
        assert ref.sizes(m, nc, f)[1] >= nc


def test_python_params_routing():
    from raft_b200.cluster import KMeansParams
    assert KMeansParams(n_clusters=3).oversampling_factor is None
    assert KMeansParams(n_clusters=3, oversampling_factor=0).oversampling_factor == 0.0
    assert KMeansParams(n_clusters=3, oversampling_factor=2).oversampling_factor == 2.0
    for bad in (-1.0, float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError):
            KMeansParams(n_clusters=3, oversampling_factor=bad)
    import pylibraft.cluster.kmeans as pk
    from raft_b200.cluster import init_scalable
    assert pk.init_scalable is init_scalable


def test_model_draw_law():
    """ES keys: the first of n draws is distributed ~ p, and zero mass is never drawn while mass remains."""
    rng = np.random.default_rng(0)
    p = np.array([0.0, 1.0, 2.0, 3.0, 0.0, 4.0])
    first = np.bincount([ref.es_draw(p, 1, rng)[0] for _ in range(20000)], minlength=6) / 20000
    np.testing.assert_allclose(first, p / p.sum(), atol=0.015)
    for _ in range(100):
        assert set(ref.es_draw(p, 4, rng)) == {1, 2, 3, 5}
    assert list(ref.es_draw(np.array([1.0, np.nan, 0.0]), 3, rng)) == [0, 2, 1]   # +inf before NaN


def test_model_candidates():
    x, _, _ = kmeans_ref.blobs(3000, 8, 10, seed=3, spread=0.3)
    ids, W = ref.candidates(x, 10, 2.0, seed=1)
    assert len(ids) == ref.sizes(3000, 10, 2.0)[1] and len(set(ids)) == len(ids)
    assert W.sum() == 3000


@pytest.mark.parametrize("nc,k", [(12, 16), (50, 32)])
def test_model_cost_against_greedy(nc, k):
    """On blobs of spread 0.3 (20000 rows) the model's seeding cost is 0.48-0.65 of greedy k-means++'s over six seeds
    and n_clusters = 12, 20, 50.  The converged inertia of a single seed varies more (0.84-1.21 of the greedy-seeded
    fit's), its mean over six seeds is 0.93-1.01 of greedy's."""
    x, _, _ = kmeans_ref.blobs(20000, k, nc, seed=nc + k, spread=0.3)
    fa = fb = 0.0
    for s in range(3):
        a = ref.init_scalable(x, nc, 2.0, seed=s)
        b = ref.greedy_plus_plus(x, nc, seed=s)
        assert kmeans_ref.cost(x, a) < 0.7 * kmeans_ref.cost(x, b)
        fa += kmeans_ref.lloyd(x, a, 300, 1e-4)[2]
        fb += kmeans_ref.lloyd(x, b, 300, 1e-4)[2]
    assert fa < 1.1 * fb
