"""single_linkage without a GPU: the fp64 reference (tests/single_linkage_ref.py) against scipy's single linkage and
minimum spanning tree, the ABI declarations, the workspace queries and the argument checks of the C ABI."""
import ctypes
import os
import re

import numpy as np
import pytest

import single_linkage_ref as ref
from raft_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
NEW = ["b2d_mst_workspace_bytes", "b2d_mst", "b2d_single_linkage_workspace_bytes", "b2d_single_linkage",
       "b2d_debug_single_linkage_plan"]
L2, L2SQRT, COSINE = 0, 1, 2


@pytest.mark.parametrize("m,d", [(2, 3), (9, 2), (40, 5), (64, 16)])
def test_reference_equals_scipy_on_complete_graphs(m, d):
    hierarchy = pytest.importorskip("scipy.cluster.hierarchy")
    x = np.random.default_rng(m + d).standard_normal((m, d))
    Z = hierarchy.linkage(x, method="single", metric="euclidean")
    for nc in sorted({1, 2, m // 3 + 1, m}):
        ch, de, sz, lab, ncomp = ref.single_linkage(x, nc, c=m)   # n_nb = m: the complete graph
        assert ncomp == 1
        assert (ch == Z[:, :2]).all() and (sz == Z[:, 3]).all()
        np.testing.assert_allclose(de, Z[:, 2], rtol=1e-12)
        want = hierarchy.fcluster(Z, nc, criterion="maxclust")
        assert (lab == ref.canonical_labels(want)).all()
        assert lab.max() == nc - 1


def test_reference_connects_components():
    """Two far groups with n_nb below their size: the kNN graph has several components and the connecting edge of the
    groups is the exact nearest pair."""
    hierarchy = pytest.importorskip("scipy.cluster.hierarchy")
    rng = np.random.default_rng(4)
    x = np.concatenate([rng.standard_normal((30, 3)), 50 + rng.standard_normal((30, 3))])
    ch, de, sz, lab, ncomp = ref.single_linkage(x, 2, c=1)   # n_nb = 5
    assert ncomp >= 2
    Z = hierarchy.linkage(x, method="single")
    np.testing.assert_allclose(de[-1], Z[-1, 2], rtol=1e-12)
    assert (lab == np.repeat([0, 1], 30)).all() and sz[-1] == 60


@pytest.mark.parametrize("n,e,seed", [(10, 30, 0), (200, 600, 1), (500, 400, 2)])
def test_kruskal_equals_scipy_minimum_spanning_tree(n, e, seed):
    csgraph = pytest.importorskip("scipy.sparse.csgraph")
    rng = np.random.default_rng(seed)
    src, dst = rng.integers(0, n, e), rng.integers(0, n, e)
    w = rng.uniform(1, 2, e)
    chosen, colour = ref.kruskal(src, dst, w, n)
    dense = np.full((n, n), np.inf)
    for a, b, v in zip(src, dst, w):   # scipy takes one weight per pair: the smallest
        if a != b:
            i, j = min(a, b), max(a, b)
            dense[i, j] = min(dense[i, j], v)
    dense[np.isinf(dense)] = 0
    T = csgraph.minimum_spanning_tree(dense).tocoo()
    assert sorted(zip(T.row, T.col)) == sorted((min(src[c], dst[c]), max(src[c], dst[c])) for c in chosen)
    np.testing.assert_allclose(w[chosen].sum(), T.data.sum(), rtol=1e-12)
    n_comp, lab = csgraph.connected_components(dense, directed=False)
    assert len(np.unique(colour)) == n_comp and (ref.canonical_labels(lab) == ref.canonical_labels(colour)).all()


def test_reference_tie_order():
    # equal weights: the earlier edge wins; float32 weights order -0.0 before +0.0 (the device's ordered bits)
    chosen, _ = ref.kruskal(np.array([0, 1, 0]), np.array([1, 2, 2]), np.float32([1, 1, 1]), 3)
    assert chosen.tolist() == [0, 1]
    chosen, _ = ref.kruskal(np.array([0, 0]), np.array([1, 1]), np.float32([0.0, -0.0]), 2)
    assert chosen.tolist() == [1]
    assert ref.n_neighbors(1) == 1 and ref.n_neighbors(2) == 2 and ref.n_neighbors(10 ** 6) == 34


def test_connect_tie_goes_to_the_first_tree_by_smallest_row():
    """Tree {2} (x = 0) has two nearest rows at squared distance 25: row 1 (tree {1}) and row 3 (tree {0, 3}).  The
    smaller row is 1; the first in (smallest row of its tree, row) order is 3, and that one wins."""
    x = np.array([[100.0], [5.0], [0.0], [-5.0]])
    colour = np.array([0, 1, 2, 0])
    src, dst, w = ref.connect_edges(x, colour)
    assert src.tolist() == [3, 1, 2] and dst.tolist() == [2, 2, 3] and w.tolist() == [25, 25, 25]


def sl_plan(m, comps):
    """b2d_debug_single_linkage_plan: (chunk rows, chunks, sort block rows, sort blocks)."""
    out = (ctypes.c_int64 * 4)()
    _lib.check(_lib.lib().b2d_debug_single_linkage_plan(m, comps, ctypes.addressof(out)))
    return tuple(out)


def plan_model(m, c):
    """The plan restated: chunk rows max(128, floor(128 m / c) rounded down to 128), capped at m rounded up to 128 and
    at 2^40 / m rounded down to 128 (never below 128); sort blocks of 2048 rows, widened in steps of 2048 when
    c x blocks would pass 2^24 histogram words."""
    cap = max(128, (2 ** 40 // m) // 128 * 128)
    rows = min(max(128, (128 * m // c) // 128 * 128), -(-m // 128) * 128, cap)
    rb = 2048
    if c * -(-m // 2048) > 2 ** 24:
        nblk = max(1, 2 ** 24 // c)
        rb = -(-(-(-m // nblk)) // 2048) * 2048
    return rows, -(-m // rows), rb, -(-m // rb)


@pytest.mark.parametrize("m,comps,want", [
    (5000, 2, (5120, 1, 2048, 3)),            # one chunk: 128 m / c is past m rounded up to 128
    (5000, 125, (5120, 1, 2048, 3)),          # the last single chunk (m = 39 x 128 + 8) ...
    (5000, 126, (4992, 2, 2048, 3)),          # ... and the first split into two
    (5000, 128, (4992, 2, 2048, 3)),
    (5000, 257, (2432, 3, 2048, 3)),
    (5000, 1000, (640, 8, 2048, 3)),
    (5000, 2500, (256, 20, 2048, 3)),         # two-row trees: 256-row chunks
    (5000, 5000, (128, 40, 2048, 3)),
    (2047, 2, (2048, 1, 2048, 1)), (2048, 2, (2048, 1, 2048, 1)), (2049, 2, (2176, 1, 2048, 2)),
    (6145, 3, (6272, 1, 2048, 4)),
    (270000, 135000, (256, 1055, 4096, 66)),  # past the histogram cap: 135000 x 132 blocks > 2^24 words
    (2 ** 29, 2, (2048, 2 ** 18, 2048, 2 ** 18)),   # chunks capped at 2^40 / m rows
])
def test_single_linkage_plan(m, comps, want):
    assert sl_plan(m, comps) == want == plan_model(m, comps)


def test_single_linkage_plan_model_and_arguments():
    rng = np.random.default_rng(7)
    for m in list(rng.integers(2, 10 ** 6, 40)) + [2, 3, 127, 128, 129, 2 ** 30 - 1]:
        m = int(m)
        for c in {2, m, int(rng.integers(2, m + 1)), max(2, m // 2), max(2, m // 128)}:
            assert sl_plan(m, c) == plan_model(m, c), (m, c)
    L = _lib.lib()
    out = (ctypes.c_int64 * 4)()
    for m, c in ((1, 1), (100, 1), (100, 101), (2 ** 30, 2)):
        assert L.b2d_debug_single_linkage_plan(m, c, ctypes.addressof(out)) == _lib.B2D_ERR_INVALID_ARG, (m, c)
    assert L.b2d_debug_single_linkage_plan(100, 2, None) == _lib.B2D_ERR_INVALID_ARG


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(_lib.lib(), s)


def test_workspace_queries():
    L = _lib.lib()
    assert L.b2d_single_linkage_workspace_bytes(-1, 8, 15) == SIZE_MAX
    assert L.b2d_single_linkage_workspace_bytes(10, -1, 15) == SIZE_MAX
    assert L.b2d_single_linkage_workspace_bytes(1000, 8, 60) == SIZE_MAX    # n_nb = 69
    assert L.b2d_single_linkage_workspace_bytes(2 ** 30, 8, 15) == SIZE_MAX
    assert L.b2d_mst_workspace_bytes(-1, 5) == SIZE_MAX and L.b2d_mst_workspace_bytes(5, -1) == SIZE_MAX
    prev = 0
    for m in (1, 100, 5000, 100000, 10 ** 6):
        b = L.b2d_single_linkage_workspace_bytes(m, 32, 15)
        assert b % 1024 == 0 and b > prev
        prev = b
    # the workspace depends on (m, d, n_nb) only
    assert L.b2d_single_linkage_workspace_bytes(100, 8, 200) == L.b2d_single_linkage_workspace_bytes(100, 8, 100)


def sl(metric=L2SQRT, x=P, ldx=8, m=100, d=8, c=15, nc=4, ch=P, de=P, sz=P, lab=P, ncomp=P, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_single_linkage(None, metric, x, ldx, m, d, c, nc, ch, de, sz, lab, ncomp, ws, wsb)


@pytest.mark.parametrize("kw,rc", [
    (dict(metric=COSINE), _lib.B2D_ERR_UNSUPPORTED), (dict(metric=3), _lib.B2D_ERR_UNSUPPORTED),
    (dict(nc=0), _lib.B2D_ERR_INVALID_ARG), (dict(nc=101), _lib.B2D_ERR_INVALID_ARG),
    (dict(c=60), _lib.B2D_ERR_UNSUPPORTED), (dict(d=321, ldx=321), _lib.B2D_ERR_UNSUPPORTED),
    (dict(m=0), _lib.B2D_ERR_INVALID_ARG), (dict(d=0), _lib.B2D_ERR_INVALID_ARG),
    (dict(m=2 ** 30), _lib.B2D_ERR_UNSUPPORTED), (dict(m=2 ** 29, nc=1), _lib.B2D_ERR_UNSUPPORTED),
    (dict(ldx=7), _lib.B2D_ERR_INVALID_ARG), (dict(x=None), _lib.B2D_ERR_INVALID_ARG),
    (dict(lab=None), _lib.B2D_ERR_INVALID_ARG), (dict(ch=None), _lib.B2D_ERR_INVALID_ARG),
    (dict(ncomp=None), _lib.B2D_ERR_INVALID_ARG),
])
def test_single_linkage_invalid_arguments(kw, rc):
    assert sl(**kw) == rc, kw


def test_single_linkage_error_messages():
    L = _lib.lib()
    assert sl(c=60) == _lib.B2D_ERR_UNSUPPORTED
    msg = L.b2d_last_error().decode()
    assert "lower c (60)" in msg and "= 66 neighbours" in msg
    need = L.b2d_single_linkage_workspace_bytes(100, 8, 15)
    assert sl(ws=None, wsb=need) == _lib.B2D_ERR_WORKSPACE
    assert sl(wsb=need - 1) == _lib.B2D_ERR_WORKSPACE
    assert sl(ws=P * 256 + 8, wsb=need) == _lib.B2D_ERR_INVALID_ARG


def mst(src=P, dst=P, w=P, n=10, e=20, osrc=P, odst=P, ow=P, col=P, cnt=P, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_mst(None, src, dst, w, n, e, osrc, odst, ow, col, cnt, ws, wsb)


@pytest.mark.parametrize("kw,rc", [
    (dict(n=-1), _lib.B2D_ERR_INVALID_ARG), (dict(e=-1), _lib.B2D_ERR_INVALID_ARG),
    (dict(n=2 ** 30), _lib.B2D_ERR_UNSUPPORTED), (dict(e=2 ** 32 - 1), _lib.B2D_ERR_UNSUPPORTED),
    (dict(src=None), _lib.B2D_ERR_INVALID_ARG), (dict(w=None), _lib.B2D_ERR_INVALID_ARG),
    (dict(cnt=None), _lib.B2D_ERR_INVALID_ARG), (dict(col=None), _lib.B2D_ERR_INVALID_ARG),
    (dict(osrc=None), _lib.B2D_ERR_INVALID_ARG), (dict(ws=None, wsb=64), _lib.B2D_ERR_WORKSPACE),
])
def test_mst_invalid_arguments(kw, rc):
    assert mst(**kw) == rc, kw


def test_python_api():
    from raft_b200.cluster import LinkageOutput, mst, single_linkage
    import pylibraft.cluster.single_linkage as pl
    assert pl.single_linkage is single_linkage and pl.mst is mst
    assert LinkageOutput._fields == ("children", "deltas", "sizes", "labels", "n_connected_components")
