"""kmeans without a GPU: the fp64 reference (tests/kmeans_ref.py) against scikit-learn, the ABI declarations, the
workspace query and the argument checks of the C ABI."""
import os
import re

import numpy as np
import pytest

import kmeans_ref
from raft_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
NEW = ["b2d_kmeans_workspace_bytes", "b2d_kmeans_fit", "b2d_kmeans_predict", "b2d_kmeans_update_centroids",
       "b2d_kmeans_init_plus_plus"]


@pytest.mark.parametrize("k,nc", [(2, 3), (16, 8), (5, 20)])
def test_reference_matches_sklearn_lloyd(k, nc):
    cl = pytest.importorskip("sklearn.cluster")
    x, _, _ = kmeans_ref.blobs(600, k, nc, seed=k + nc, spread=0.2)
    x = x.astype(np.float64)
    c0 = x[:: len(x) // nc][:nc].astype(np.float32)
    for max_iter in (1, 3, 50):
        c, lab, inertia, _ = kmeans_ref.lloyd(x, c0, max_iter, 0.0)
        assert np.bincount(lab, minlength=nc).min() > 0   # sklearn relocates empty clusters: not compared
        sk = cl.KMeans(n_clusters=nc, init=c0.astype(np.float64), n_init=1, max_iter=max_iter, tol=0,
                       algorithm="lloyd").fit(x)
        np.testing.assert_allclose(c, sk.cluster_centers_, rtol=1e-5, atol=1e-5)
        assert (lab == sk.predict(x)).all()
        np.testing.assert_allclose(inertia, sk.inertia_, rtol=1e-6)


def test_reference_update_rules():
    x = np.arange(12, dtype=np.float32).reshape(6, 2)
    old = np.full((4, 2), 7.25, np.float32)
    lab = np.array([0, 0, 1, -1, 4, 1])
    w = np.array([1, 3, 2, 5, 5, 0], np.float32)
    new, W = kmeans_ref.update(x, lab, old, w)
    np.testing.assert_array_equal(new[0], np.float32([(0 + 3 * 2) / 4, (1 + 3 * 3) / 4]))
    np.testing.assert_array_equal(new[1], x[2])                  # the zero-weight row adds nothing
    assert (new[2:] == old[2:]).all()                             # empty clusters keep their bits
    np.testing.assert_array_equal(W, np.float32([4, 2, 0, 0]))   # out-of-range labels are skipped


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(_lib.lib(), s)
    assert (_lib.B2D_KMEANS_INIT_PLUS_PLUS, _lib.B2D_KMEANS_INIT_RANDOM, _lib.B2D_KMEANS_INIT_ARRAY) == (0, 1, 2)


def test_workspace_query():
    L = _lib.lib()
    assert L.b2d_kmeans_workspace_bytes(-1, 8, 2) == SIZE_MAX
    assert L.b2d_kmeans_workspace_bytes(10, -1, 2) == SIZE_MAX
    assert L.b2d_kmeans_workspace_bytes(10, 8, -1) == SIZE_MAX
    prev = 0
    for m in (1, 100, 5000, 100000):
        b = L.b2d_kmeans_workspace_bytes(m, 32, 1)
        assert b % 1024 == 0 and b > prev
        prev = b
    # the histogram is capped: 10^6 rows and 10^5 clusters stay far below n_clusters x m words
    assert L.b2d_kmeans_workspace_bytes(10 ** 6, 128, 10 ** 5) < 2 * 10 ** 9


def fit(nc=4, max_iter=10, tol=1e-4, init=2, n_init=1, x=P, ldx=8, w=None, m=100, k=8, c=P, inertia=P, n_iter=P,
        ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_kmeans_fit(None, nc, max_iter, tol, init, n_init, 0, 0, x, ldx, w, m, k, c, inertia, n_iter, ws,
                                     wsb)


@pytest.mark.parametrize("kw", [dict(nc=0), dict(nc=101), dict(k=0), dict(ldx=7), dict(x=None), dict(c=None),
                                dict(inertia=None), dict(n_iter=None), dict(max_iter=-1), dict(tol=-1.0),
                                dict(tol=float("nan")), dict(init=3), dict(n_init=0), dict(m=2 ** 31)])
def test_fit_invalid_arguments(kw):
    assert fit(**kw) == _lib.B2D_ERR_INVALID_ARG, kw


def test_workspace_errors_and_empty_input():
    need = _lib.lib().b2d_kmeans_workspace_bytes(100, 8, 4)
    assert fit(ws=None, wsb=need) == _lib.B2D_ERR_WORKSPACE
    assert fit(wsb=need - 1) == _lib.B2D_ERR_WORKSPACE
    assert fit(ws=P * 256 + 8, wsb=need) == _lib.B2D_ERR_INVALID_ARG   # not 256-byte aligned
    assert fit(m=0, nc=0, x=None, c=None) == _lib.B2D_OK
    L = _lib.lib()
    assert L.b2d_kmeans_predict(None, P, 8, None, 100, 8, P, 101, None, None, 1, P * 256, 1 << 40) == _lib.B2D_ERR_INVALID_ARG
    assert L.b2d_kmeans_update_centroids(None, P, 8, None, None, 100, 8, P, 4, P, None, P * 256, 1 << 40) == \
        _lib.B2D_ERR_INVALID_ARG
    assert L.b2d_kmeans_init_plus_plus(None, P, 8, None, 100, 8, 0, 0, P, P * 256, 1 << 40) == _lib.B2D_ERR_INVALID_ARG
    assert L.b2d_kmeans_predict(None, P, 8, None, 0, 8, P, 4, None, None, 1, None, 0) == _lib.B2D_OK


def test_python_params():
    from raft_b200.cluster import KMeansParams
    p = KMeansParams(n_clusters=3, oversampling_factor=2.0, batch_samples=1 << 15, batch_centroids=0, verbosity=4)
    assert p.init_method == "KMeansPlusPlus" and p.n_init == 1 and p.max_iter == 300 and p.tol == 1e-4
    with pytest.raises(_lib.LogicError):
        KMeansParams(n_clusters=3, metric="cosine")
    import pylibraft.cluster.kmeans as pk
    assert pk.fit is not None and pk.KMeansParams is KMeansParams
