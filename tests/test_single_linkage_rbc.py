"""Exact single linkage on the random ball cover without a GPU: the oracle (tests/emst_ref.py) against
scipy.cluster.hierarchy.linkage(method="single") and against single_linkage_ref.kruskal, the ABI declarations, every
argument check of b2d_emst_rbc and b2d_single_linkage_rbc with its status and message, B2D_ERR_CUDA without a device,
the recorded workspace contract (tests/golden/single_linkage_rbc_workspace_contract.json) and the Python argument
errors.  The C++ shim is in tests/test_single_linkage_rbc_shim.py, the GPU tier in tests/test_single_linkage_rbc_gpu.py."""
import os
import re

import numpy as np
import pytest
import torch

import emst_ref
from single_linkage_ref import canonical_labels, kruskal
from raft_b200 import _lib
from test_workspace_contract import SIZE_MAX, load, replay_bytes, replay_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE
L2, L2SQRT = 4, 5   # L2Unexpanded, L2SqrtUnexpanded
NEW = ["b2d_emst_rbc_workspace_bytes", "b2d_emst_rbc", "b2d_single_linkage_rbc_workspace_bytes",
       "b2d_single_linkage_rbc"]


def L():
    return _lib.lib()


def distinct_points(m, d, seed):
    """random points whose pair values are all distinct (the first seed from `seed` on that gives them)"""
    while True:
        x = np.random.default_rng(seed).random((m, d)).astype(np.float32)
        _, _, s = emst_ref.pair_values(x)
        if len(np.unique(s)) == len(s):
            return x
        seed += 1


@pytest.mark.parametrize("metric", ["sqeuclidean", "euclidean"])
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("m", [2, 3, 17, 120])
def test_oracle_equals_scipy_single_linkage(m, d, metric):
    hierarchy = pytest.importorskip("scipy.cluster.hierarchy")
    from scipy.spatial.distance import squareform
    x = distinct_points(m, d, 100 * m + d)
    xt = torch.from_numpy(x)
    import ball_cover_ref as bref
    dd = bref.dist(xt, xt, metric).double().numpy()
    np.fill_diagonal(dd, 0)
    Z = hierarchy.linkage(squareform(dd, checks=False), method="single")
    for nc in (1, 2, max(1, m // 3), m):
        ch, de, sz, lab = emst_ref.single_linkage(x, nc, metric)
        assert (ch == Z[:, :2].astype(np.int64)).all()
        assert (sz == Z[:, 3].astype(np.int64)).all()
        np.testing.assert_allclose(de, Z[:, 2], rtol=2 ** -23, atol=0)
        want = canonical_labels(hierarchy.fcluster(Z, nc, criterion="maxclust"))
        assert (lab == want).all()


@pytest.mark.parametrize("kind", ["uniform", "lattice", "duplicates"])
def test_oracle_loop_equals_kruskal(kind):
    r = np.random.default_rng(3)
    if kind == "uniform":
        x = r.random((90, 2)).astype(np.float32)
    elif kind == "lattice":
        x = np.stack(np.meshgrid(np.arange(6), np.arange(7), indexing="ij"), -1).reshape(-1, 2).astype(np.float32)
    else:
        x = r.random((9, 3)).astype(np.float32)[r.integers(0, 9, 60)]
    src, dst, s = emst_ref.pair_values(x)
    full, colour = kruskal(src, dst, s, len(x))
    assert (colour == 0).all() and (emst_ref.kruskal_tree(src, dst, s, len(x)) == full).all()
    a, b, w = emst_ref.emst(x)
    assert (a < b).all() and (a == src[full]).all() and (b == dst[full]).all() and (w == s[full]).all()
    # the order of the tree edges is (s, min row, max row)
    assert (np.lexsort((b, a, w)) == np.arange(len(w))).all()


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(L(), s)
    assert "b2d_single_linkage(" in hdr and "b2d_mst(" in hdr


@pytest.mark.parametrize("fn", ["b2d_emst_rbc_workspace_bytes", "b2d_single_linkage_rbc_workspace_bytes"])
def test_workspace_queries(fn):
    q = getattr(L(), fn)
    for args in ((0, 2, 0), (-1, 2, 0), (2 ** 30, 2, 0), (10, 1, 0), (10, 4, 0), (10, 2, -1), (10, 2, 11)):
        assert q(*args) == SIZE_MAX, args
    for m, d in ((1, 2), (1000, 3), (10 ** 6, 2), (2 ** 30 - 1, 3)):
        full = q(m, d, 0)
        index = L().b2d_ball_cover_index_bytes(m, d, 0)
        build = L().b2d_ball_cover_build_workspace_bytes(m, d, 0)
        # the index, then the build's scratch, which the rounds' arrays (48 bytes a row and the sort's scratch) overlap
        assert full >= index + max(build, 48 * m)
        assert full <= index + max(build, 60 * m + (4 << 20))
        assert q(m, d, int(np.ceil(np.sqrt(m)))) == full
    # single linkage adds the host copies of the edges
    assert L().b2d_single_linkage_rbc_workspace_bytes(10 ** 6, 2, 0) > L().b2d_emst_rbc_workspace_bytes(10 ** 6, 2, 0)


def test_workspace_contract_bytes():
    c = load("single_linkage_rbc_workspace_contract.json")
    for fn in ("b2d_emst_rbc_workspace_bytes", "b2d_single_linkage_rbc_workspace_bytes"):
        for m, d, nl, want in replay_bytes(c, fn):
            assert (want == SIZE_MAX) == (not (1 <= m < 2 ** 30 and d in (2, 3) and 0 <= nl <= m)), (m, d, nl)


def test_workspace_contract_errors():
    assert replay_errors(load("single_linkage_rbc_workspace_contract.json")) == 2 * 2 * 2 * 3


def emst_call(metric=L2SQRT, x=P, ldx=2, m=100, d=2, nl=0, seed=1, src=P, dst=P, w=P, ws=P * 256, wsb=1 << 40):
    return L().b2d_emst_rbc(None, metric, x, ldx, m, d, nl, seed, src, dst, w, ws, wsb)


def sl_call(metric=L2SQRT, x=P, ldx=2, m=100, d=2, nl=0, seed=1, nc=3, ch=P, de=P, sz=P, lab=P, ws=P * 256,
            wsb=1 << 40):
    return L().b2d_single_linkage_rbc(None, metric, x, ldx, m, d, nl, seed, nc, ch, de, sz, lab, ws, wsb)


def metric_msg(fn, metric):
    return "%s supports the L2Unexpanded and L2SqrtUnexpanded metrics, got metric %d" % (fn, metric)


COMMON = [
    (dict(metric=0), U, "metric", 0),
    (dict(metric=1), U, "metric", 1),
    (dict(metric=-1), U, "metric", -1),
    (dict(metric=13), U, "metric", 13),
    (dict(m=0), E, "m must be positive and n_landmarks non-negative", None),
    (dict(m=-1), E, "m must be positive and n_landmarks non-negative", None),
    (dict(nl=-1), E, "m must be positive and n_landmarks non-negative", None),
    (dict(d=1, ldx=1), U, "supports d = 2 and d = 3, got d = 1", None),
    (dict(d=4, ldx=4), U, "supports d = 2 and d = 3, got d = 4", None),
    (dict(d=0), U, "supports d = 2 and d = 3, got d = 0", None),
    (dict(m=2 ** 30, nl=0), U, ": m must be below 2^30", None),
    (dict(nl=101), E, "n_landmarks must be in [0, m] (0: ceil(sqrt(m)))", None),
    (dict(x=None), E, "null x", None),
    (dict(ldx=1), E, "leading dimension smaller than d", None),
    (dict(d=3, ldx=2), E, "leading dimension smaller than d", None),
    (dict(ws=None, wsb=0), W, "workspace too small: need ", None),
    (dict(wsb=10), W, "workspace too small: need ", None),
    (dict(ws=P * 256 + 8), E, "workspace must be 256-byte aligned", None),
]


def expected(fn, msg, metric):
    if msg == "metric":
        return metric_msg(fn, metric)
    if msg.startswith("supports") or msg.startswith(":"):
        return fn + (" " if msg.startswith("supports") else "") + msg
    return msg


@pytest.mark.parametrize("kw,rc,msg,metric", COMMON + [
    (dict(src=None), E, "null out_src / out_dst / out_w", None),
    (dict(dst=None), E, "null out_src / out_dst / out_w", None),
    (dict(w=None), E, "null out_src / out_dst / out_w", None),
])
def test_emst_invalid_arguments(kw, rc, msg, metric):
    assert emst_call(**kw) == rc, kw
    assert L().b2d_last_error().decode().startswith(expected("emst rbc", msg, metric))


@pytest.mark.parametrize("kw,rc,msg,metric", COMMON + [
    (dict(nc=0), E, "n_clusters must be in [1, m]", None),
    (dict(nc=101), E, "n_clusters must be in [1, m]", None),
    (dict(ch=None), E, "null children / deltas / sizes / labels", None),
    (dict(de=None), E, "null children / deltas / sizes / labels", None),
    (dict(sz=None), E, "null children / deltas / sizes / labels", None),
    (dict(lab=None), E, "null children / deltas / sizes / labels", None),
])
def test_single_linkage_invalid_arguments(kw, rc, msg, metric):
    assert sl_call(**kw) == rc, kw
    assert L().b2d_last_error().decode().startswith(expected("single_linkage rbc", msg, metric))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert emst_call() == _lib.B2D_ERR_CUDA
    assert emst_call(m=1, src=None, dst=None, w=None) == _lib.B2D_ERR_CUDA   # one row: no outputs, the index still
    assert emst_call(d=3, ldx=5, metric=L2) == _lib.B2D_ERR_CUDA
    assert sl_call() == _lib.B2D_ERR_CUDA
    assert sl_call(m=1, nc=1, ch=None, de=None, sz=None) == _lib.B2D_ERR_CUDA


class FakeCuda:
    """an object with a __cuda_array_interface__ that is never read (the calls below fail in validation)"""

    def __init__(self, shape, typestr="<f4", strides=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (P, False), "version": 3,
                                         "strides": strides}


PY_ERRORS = [
    (dict(metric="cosine"), _lib.LogicError, "supports the euclidean and sqeuclidean metrics"),
    (dict(metric="manhattan"), _lib.LogicError, "supports the euclidean and sqeuclidean metrics"),
    (dict(shape=(10, 4)), _lib.LogicError, "supports d = 2 and d = 3, got d = 4"),
    (dict(shape=(10, 1)), _lib.LogicError, "supports d = 2 and d = 3, got d = 1"),
    (dict(n_landmarks=11), _lib.LogicError, "n_landmarks must be in [0, m]"),
    (dict(n_landmarks=-1), _lib.LogicError, "n_landmarks must be in [0, m]"),
    (dict(strides=(8, 8)), ValueError, "X must have contiguous rows"),
    (dict(strides=(4, 4)), ValueError, "row pitch of at least d elements"),
]


@pytest.mark.parametrize("kw,exc,msg", PY_ERRORS + [
    (dict(linkage="ward"), _lib.LogicError, "linkage must be 'knn_graph' or 'pairwise'"),
])
def test_python_single_linkage_argument_errors(kw, exc, msg):
    from raft_b200.cluster import single_linkage
    kw = dict(kw)
    x = FakeCuda(kw.pop("shape", (10, 2)), strides=kw.pop("strides", None))
    args = dict(linkage="pairwise")
    args.update(kw)
    with pytest.raises(exc, match=re.escape(msg)):
        single_linkage(x, 2, handle=object(), **args)


@pytest.mark.parametrize("kw,exc,msg", PY_ERRORS)
def test_python_emst_argument_errors(kw, exc, msg):
    from raft_b200.cluster import emst
    kw = dict(kw)
    x = FakeCuda(kw.pop("shape", (10, 2)), strides=kw.pop("strides", None))
    with pytest.raises(exc, match=re.escape(msg)):
        emst(x, handle=object(), **kw)


def test_python_signatures():
    import inspect
    from raft_b200.cluster import emst, single_linkage
    import pylibraft.cluster.single_linkage as pl
    params = list(inspect.signature(single_linkage).parameters.items())
    assert [(k, p.default) for k, p in params[2:]] == [
        ("metric", "euclidean"), ("c", 15), ("linkage", "knn_graph"), ("n_landmarks", None), ("seed", 0),
        ("handle", None)]
    params = list(inspect.signature(emst).parameters.items())
    assert [(k, p.default) for k, p in params[1:]] == [
        ("metric", "euclidean"), ("n_landmarks", None), ("seed", 0), ("handle", None)]
    assert pl.emst is emst and pl.single_linkage is single_linkage
