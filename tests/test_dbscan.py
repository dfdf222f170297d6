"""DBSCAN without a GPU: the reference (tests/dbscan_ref.py) against sklearn.cluster.DBSCAN on symmetric adjacency and
against scipy's connected components on asymmetric adjacency, the ABI declarations, the workspace queries and the
argument checks of the C ABI.  The workspace contract (tests/golden/dbscan_workspace_contract.json) is replayed by
tests/test_workspace_contract.py."""
import os
import re

import numpy as np
import pytest

from dbscan_ref import dbscan_ref
from raft_b200 import _lib
from test_workspace_contract import SIZE_MAX

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
NEW = ["b2d_dbscan_workspace_bytes", "b2d_dbscan_fit"]
L2, L2SQRT, COSINE = 0, 1, 2


def random_adjacency(m, density, seed, symmetric):
    rng = np.random.default_rng(seed)
    A = rng.random((m, m)) < density
    if symmetric:
        A = np.triu(A, 1)
        A = A | A.T
    np.fill_diagonal(A, True)
    return A


@pytest.mark.parametrize("m", [1, 7, 60, 200])
@pytest.mark.parametrize("density", [0.0, 0.01, 0.05, 0.3])
def test_reference_equals_sklearn(m, density):
    cluster = pytest.importorskip("sklearn.cluster")
    A = random_adjacency(m, density, m * 100 + int(density * 100), True)
    D = np.where(A, 0.5, 2.0)
    np.fill_diagonal(D, 0.0)
    for ms in (1, 2, 5, m + 1):
        sk = cluster.DBSCAN(eps=1.0, min_samples=ms, metric="precomputed").fit(D)
        lab, csi, nc = dbscan_ref(A, ms)
        assert (lab == sk.labels_).all(), (m, density, ms)
        ncore = len(sk.core_sample_indices_)
        assert (csi[:ncore] == sk.core_sample_indices_).all() and (csi[ncore:] == -1).all()
        assert nc == len(set(sk.labels_) - {-1})


def components_construction(A, min_samples):
    """The same rules built another way: scipy's components of the core subgraph of A | A^T, renumbered by smallest
    row, and the border rule over the columns."""
    csgraph = pytest.importorskip("scipy.sparse.csgraph")
    m = A.shape[0]
    core = A.sum(axis=0) >= min_samples
    cidx = np.flatnonzero(core)
    labels = np.full(m, -1, np.int64)
    if cidx.size:
        sub = A[np.ix_(cidx, cidx)]
        _, comp = csgraph.connected_components(sub | sub.T, directed=False)
        first = {}
        for c in comp:
            first.setdefault(c, len(first))
        labels[cidx] = [first[c] for c in comp]
        for b in np.flatnonzero(~core):
            hit = A[b] & core
            if hit.any():
                labels[b] = labels[hit].min()
    return labels, cidx, len(set(labels[cidx].tolist()))


@pytest.mark.parametrize("m,density", [(30, 0.05), (150, 0.01), (150, 0.04), (300, 0.005)])
def test_reference_on_asymmetric_adjacency(m, density):
    A = random_adjacency(m, density, m + int(1000 * density), False)
    assert not (A == A.T).all()
    for ms in (1, 2, 3, 5, m + 1):
        lab, csi, nc = dbscan_ref(A, ms)
        want, cidx, wnc = components_construction(A, ms)
        assert (lab == want).all() and nc == wnc
        assert (csi[:cidx.size] == cidx).all() and (csi[cidx.size:] == -1).all()


@pytest.mark.parametrize("m,density,symmetric", [(1, 0.0, True), (80, 0.03, False), (250, 0.01, True), (400, 0.004, False)])
def test_edge_list_reference_equals_dense(m, density, symmetric):
    pytest.importorskip("scipy.sparse.csgraph")
    from dbscan_ref import dbscan_ref_edges
    A = random_adjacency(m, density, 7 * m, symmetric)
    rows, cols = np.nonzero(A)
    for ms in (1, 2, 4, m + 1):
        want = dbscan_ref(A, ms)
        got = dbscan_ref_edges(rows, cols, m, ms)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all() and got[2] == want[2]


def test_reference_uses_columns():
    # A[0, 1] and A[0, 2] set: columns 1 and 2 have degree 2 (core at min_samples 2), column 0 degree 1.  Cores 1 and 2
    # are not linked (A[1, 2] = A[2, 1] = 0): two clusters, and row 0 takes the smaller one
    A = np.eye(3, dtype=bool)
    A[0, 1] = A[0, 2] = True
    lab, csi, nc = dbscan_ref(A, 2)
    assert lab.tolist() == [0, 0, 1] and csi.tolist() == [1, 2, -1] and nc == 2
    # the transpose: row 0 is core (degree 3) and links both; rows 1 and 2 are border points of its cluster
    lab, csi, nc = dbscan_ref(A.T, 2)
    assert lab.tolist() == [0, 0, 0] and csi.tolist() == [0, -1, -1] and nc == 1


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(_lib.lib(), s)


def test_workspace_queries():
    L = _lib.lib()
    for args in ((-1, 8, 0), (10, -1, 0), (10, 8, -1)):
        assert L.b2d_dbscan_workspace_bytes(*args) == SIZE_MAX, args
    # the batch plan: 0 means 2^30 bytes; below 256 columns per batch the batch stays 256 wide
    assert L.b2d_dbscan_workspace_bytes(10 ** 5, 32, 0) == L.b2d_dbscan_workspace_bytes(10 ** 5, 32, 1 << 30)
    assert L.b2d_dbscan_workspace_bytes(10 ** 5, 32, 1) == L.b2d_dbscan_workspace_bytes(10 ** 5, 32, 256 * 10 ** 5)
    small, big = L.b2d_dbscan_workspace_bytes(10 ** 5, 32, 1 << 26), L.b2d_dbscan_workspace_bytes(10 ** 5, 32, 1 << 30)
    assert big - small >= (1 << 30) - (1 << 26) - 10 ** 5 * 256
    assert L.b2d_dbscan_workspace_bytes(1000, 32, 0) >= 1000 * 1008   # one batch, pitch rounded up to 16


def fit(metric=L2SQRT, x=P, ldx=8, m=100, d=8, eps=0.5, ms=5, mb=0, lab=P, csi=P, ncl=P, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_dbscan_fit(None, metric, x, ldx, m, d, eps, ms, mb, lab, csi, ncl, ws, wsb)


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(metric=3), _lib.B2D_ERR_UNSUPPORTED, "dbscan supports the L2SqrtExpanded, L2Expanded and CosineExpanded metrics"),
    (dict(metric=-1), _lib.B2D_ERR_UNSUPPORTED, "dbscan supports the L2SqrtExpanded, L2Expanded and CosineExpanded metrics"),
    (dict(metric=10), _lib.B2D_ERR_UNSUPPORTED, "dbscan supports the L2SqrtExpanded, L2Expanded and CosineExpanded metrics"),
    (dict(m=-1), _lib.B2D_ERR_INVALID_ARG, "negative extent or batch size"),
    (dict(d=-1), _lib.B2D_ERR_INVALID_ARG, "negative extent or batch size"),
    (dict(mb=-1), _lib.B2D_ERR_INVALID_ARG, "negative extent or batch size"),
    (dict(m=2 ** 31), _lib.B2D_ERR_INVALID_ARG, "dbscan: m must be below 2^31"),
    (dict(d=0), _lib.B2D_ERR_INVALID_ARG, "d must be positive"),
    (dict(d=321, ldx=321), _lib.B2D_ERR_UNSUPPORTED, "dbscan supports d <= 320 (the whole distance at once)"),
    (dict(ms=0), _lib.B2D_ERR_INVALID_ARG, "min_samples must be >= 1"),
    (dict(ms=-3), _lib.B2D_ERR_INVALID_ARG, "min_samples must be >= 1"),
    (dict(x=None), _lib.B2D_ERR_INVALID_ARG, "null x / labels"),
    (dict(lab=None), _lib.B2D_ERR_INVALID_ARG, "null x / labels"),
    (dict(ldx=7), _lib.B2D_ERR_INVALID_ARG, "leading dimension smaller than d"),
    (dict(ws=None, wsb=0), _lib.B2D_ERR_WORKSPACE, "workspace too small: need "),
    (dict(ws=P * 256 + 8), _lib.B2D_ERR_INVALID_ARG, "workspace must be 256-byte aligned"),
])
def test_fit_invalid_arguments(kw, rc, msg):
    assert fit(**kw) == rc, kw
    assert _lib.lib().b2d_last_error().decode().startswith(msg)


def test_fit_empty_is_a_noop():
    # m == 0 touches nothing, whatever the pointers; NaN and negative eps are not errors (nothing is adjacent)
    assert fit(m=0, x=None, lab=None, ws=None, wsb=0) == _lib.B2D_OK


def test_python_api():
    import raft_b200.cluster as cl
    import pylibraft.cluster as plc
    assert cl.dbscan.__name__ == "dbscan" and cl.DbscanOutput._fields == ("labels", "core_sample_indices", "n_clusters")
    assert not hasattr(plc, "dbscan")
