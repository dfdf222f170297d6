"""HDBSCAN on the random ball cover without a GPU: the oracle (tests/hdbscan_ref.py) against
sklearn.cluster.HDBSCAN(metric="precomputed") on its own matrix, the host tree stage (raft_b200/csrc/hdbscan_tree.cuh,
compiled on its own) against the oracle on the oracle's edges, the ABI declarations, every argument check of
b2d_hdbscan_rbc_fit with its status and message, B2D_ERR_CUDA without a device, the recorded workspace contract
(tests/golden/hdbscan_rbc_workspace_contract.json) and the Python argument errors.  The GPU tier is in
tests/test_hdbscan_rbc_gpu.py, the C++ shim in tests/test_hdbscan_rbc_shim.py.

Equal mutual-reachability weights are common once min_samples > 2, and HDBSCAN's clusters depend on the order in which
its tree merges tied edges: the contract fixes that order as (w, min row, max row), while sklearn's follows its own
Prim pass and an unstable sort.  So the whole-fit comparison with sklearn runs where the tree's weights are distinct
(min_samples 1 and 2), and with ties sklearn's tree stages are given the oracle's ordered tree."""
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
import torch

import cpp_build
import hdbscan_ref as H
from raft_b200 import _lib
from test_workspace_contract import SIZE_MAX, load, replay_bytes, replay_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE
L2, L2SQRT = 4, 5   # L2Unexpanded, L2SqrtUnexpanded
NEW = ["b2d_hdbscan_rbc_workspace_bytes", "b2d_hdbscan_rbc_fit"]
SELECTIONS = [(method, single, eps) for method in ("eom", "leaf") for single in (False, True) for eps in (0.0, 0.2)]


def L():
    return _lib.lib()


def data(kind, m, d, seed):
    r = np.random.default_rng(seed)
    if kind == "uniform":
        return r.random((m, d), dtype=np.float32)
    if kind == "blobs":
        c = r.random((4, d)) * 6
        return (c[r.integers(0, 4, m)] + r.normal(0, 0.4, (m, d))).astype(np.float32)
    if kind == "duplicates":   # w = 0 between distinct rows: infinite lambdas
        return r.random((max(1, m // 6), d)).astype(np.float32)[r.integers(0, max(1, m // 6), m)]
    raise ValueError(kind)


def dense(x, metric):
    s = H.pair_matrix(x)
    return (np.sqrt(s, dtype=np.float32) if metric == "euclidean" else s).astype(np.float64)


@pytest.mark.parametrize("metric", ["euclidean", "sqeuclidean"])
@pytest.mark.parametrize("kind,m,d,seed", [("uniform", 150, 2, 1), ("blobs", 240, 2, 2), ("blobs", 200, 3, 3),
                                           ("uniform", 90, 3, 4)])
@pytest.mark.parametrize("mcs,ms", [(5, 1), (5, 2), (12, 2), (3, 1), (40, 2)])
def test_oracle_equals_sklearn(kind, m, d, seed, mcs, ms, metric):
    """min_samples 1 and 2: the tree's weights are distinct, so any tree order is the contract's"""
    skc = pytest.importorskip("sklearn.cluster")
    x = data(kind, m, d, seed)
    src, dst, w, _ = H.mr_tree(x, ms, metric)
    assert len(np.unique(w)) == len(w)
    D = dense(x, metric)
    for method, single, eps in SELECTIONS:
        eps = eps if metric == "euclidean" else eps * eps
        lab, prob, n = H.tree_labels(src, dst, w, m, mcs, method, single, eps)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            sk = skc.HDBSCAN(metric="precomputed", min_cluster_size=mcs, min_samples=ms, cluster_selection_epsilon=eps,
                             cluster_selection_method=method, allow_single_cluster=single, copy=True).fit(D)
        assert (H.canonical(sk.labels_) == lab).all(), (method, single, eps)
        np.testing.assert_allclose(prob, sk.probabilities_, rtol=0, atol=1e-12)
        assert n == len(set(sk.labels_.tolist()) - {-1})


@pytest.mark.parametrize("kind,m,d,seed", [("uniform", 200, 2, 5), ("blobs", 300, 3, 6), ("duplicates", 120, 2, 7)])
@pytest.mark.parametrize("mcs,ms", [(5, 5), (10, 3), (4, 8), (25, 10)])
def test_tree_stages_equal_sklearn_on_the_ordered_tree(kind, m, d, seed, mcs, ms):
    """with ties: sklearn's single-linkage and tree stages on the oracle's tree, taken in the contract's order, and the
    tree's weights as a multiset equal to those of sklearn's own tree"""
    pytest.importorskip("sklearn.cluster")
    from sklearn.cluster._hdbscan._linkage import MST_edge_dtype, make_single_linkage
    from sklearn.cluster._hdbscan._tree import tree_to_labels
    from sklearn.cluster._hdbscan.hdbscan import _hdbscan_brute
    x = data(kind, m, d, seed)
    src, dst, w, core = H.mr_tree(x, ms, "euclidean")
    slt = _hdbscan_brute(dense(x, "euclidean"), min_samples=ms, alpha=1.0, metric="precomputed")
    assert (np.sort(slt["value"]) == np.sort(w.astype(np.float64))).all()
    mst = np.rec.fromarrays([src.astype(np.int64), dst.astype(np.int64), w.astype(np.float64)], dtype=MST_edge_dtype)
    tree = make_single_linkage(mst)
    for method, single, eps in SELECTIONS:
        lab, prob, n = H.tree_labels(src, dst, w, m, mcs, method, single, eps)
        sl, sp = tree_to_labels(tree, mcs, method, single, eps)
        assert (H.canonical(sl) == lab).all(), (method, single, eps)
        np.testing.assert_allclose(prob, sp, rtol=0, atol=1e-12)
        assert n == len(set(sl.tolist()) - {-1})


def test_core_distances_and_prim_tree():
    """the oracle's pieces: core distances against a full sort, and its Prim tree against Kruskal in the same order"""
    from single_linkage_ref import _find
    x = data("blobs", 80, 2, 9)
    s = H.pair_matrix(x)
    for ms in (1, 2, 7):
        src, dst, w, core = H.mr_tree(x, ms)
        assert (core == np.sort(s, axis=1)[:, ms - 1]).all()
        wm = np.maximum(np.maximum(core[:, None], core[None, :]), s)
        i, j = np.triu_indices(len(x), 1)
        order = np.lexsort((j, i, wm[i, j]))
        p, chosen = list(range(len(x))), []
        for e in order:
            a, b = _find(p, int(i[e])), _find(p, int(j[e]))
            if a != b:
                p[max(a, b)] = min(a, b)
                chosen.append(e)
        assert (src == i[chosen]).all() and (dst == j[chosen]).all() and (w == wm[i, j][chosen]).all()


@pytest.fixture(scope="module")
def tree_exe(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("hdbscan_tree"))
    return cpp_build.build("hdbscan_tree_test.cu", os.path.join(d, "hdbscan_tree_test"), standalone=True), d


def host_tree(tree_exe, cases):
    """runs the host tree stage on [(src, dst, w, m, mcs, method, single, eps)]: [(labels, prob, n)]"""
    exe, d = tree_exe
    inp, out = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(inp, "wb") as f:
        for src, dst, w, m, mcs, method, single, eps in cases:
            f.write(np.array([m, mcs, method == "leaf", single], np.int64).tobytes() + np.float64(eps).tobytes())
            f.write(np.asarray(src, np.int32).tobytes() + np.asarray(dst, np.int32).tobytes() +
                    np.asarray(w, np.float32).tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw, at, got = np.fromfile(out, np.uint8), 0, []
    for c in cases:
        m = c[3]
        n = int(raw[at:at + 4].view(np.int32)[0])
        lab = raw[at + 4:at + 4 + 4 * m].view(np.int32)
        prob = raw[at + 4 + 4 * m:at + 4 + 8 * m].view(np.float32)
        got.append((lab, prob, n))
        at += 4 + 8 * m
    assert at == len(raw)
    return got


@pytest.mark.parametrize("kind,m,d", [("uniform", 300, 2), ("blobs", 500, 3), ("duplicates", 240, 2),
                                      ("duplicates", 60, 3), ("uniform", 7, 2), ("uniform", 2, 2), ("uniform", 1, 3),
                                      ("blobs", 2000, 2)])
def test_host_tree_stage_equals_oracle(tree_exe, kind, m, d):
    """exact labels, probabilities (the oracle's fp64, rounded to fp32) and counts, including infinite lambdas
    (duplicates) and all-noise fits (m below min_cluster_size, or no split)"""
    x = data(kind, m, d, 100 + m)
    cases, want = [], []
    for ms in sorted({1, min(m, 4), min(m, 11)}):
        for metric in ("euclidean", "sqeuclidean"):
            src, dst, w, _ = H.mr_tree(x, ms, metric)
            for mcs in (2, 5, 30, max(2, m + 1)):
                for method, single, eps in SELECTIONS + [("eom", True, 1e30), ("leaf", False, 1e-30)]:
                    cases.append((src, dst, w, m, mcs, method, single, eps))
                    lab, prob, n = H.tree_labels(src, dst, w, m, mcs, method, single, eps)
                    want.append((lab, prob.astype(np.float32), n))
    for (gl, gp, gn), (wl, wp, wn), c in zip(host_tree(tree_exe, cases), want, cases):
        assert gl.tobytes() == wl.tobytes(), c[3:]
        assert gp.tobytes() == wp.tobytes(), c[3:]
        assert gn == wn, c[3:]
    if kind == "duplicates":
        assert any((np.asarray(c[2]) == 0).any() for c in cases)   # infinite lambdas


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(L(), s)
    assert "#define B2D_HDBSCAN_EOM 0" in hdr and "#define B2D_HDBSCAN_LEAF 1" in hdr


def test_workspace_query():
    q = L().b2d_hdbscan_rbc_workspace_bytes
    for args in ((0, 2, 0), (-1, 2, 0), (2 ** 30, 2, 0), (10, 1, 0), (10, 4, 0), (10, 2, -1), (10, 2, 11)):
        assert q(*args) == SIZE_MAX, args
    for m, d in ((1, 2), (1000, 3), (10 ** 6, 2)):
        # the EMST's workspace plus the core distances (4 bytes a row) and one float a ball
        nl = int(np.ceil(np.sqrt(m)))
        assert q(m, d, 0) >= L().b2d_emst_rbc_workspace_bytes(m, d, 0)
        assert q(m, d, 0) <= L().b2d_emst_rbc_workspace_bytes(m, d, 0) + 4 * m + 4 * nl + 512
        assert q(m, d, nl) == q(m, d, 0)


def test_workspace_contract_bytes():
    c = load("hdbscan_rbc_workspace_contract.json")
    for m, d, nl, want in replay_bytes(c, "b2d_hdbscan_rbc_workspace_bytes"):
        assert (want == SIZE_MAX) == (not (1 <= m < 2 ** 30 and d in (2, 3) and 0 <= nl <= m)), (m, d, nl)


def test_workspace_contract_errors():
    assert replay_errors(load("hdbscan_rbc_workspace_contract.json")) == 2 * 2 * 2 * 3


def fit(metric=L2SQRT, x=P, ldx=2, m=100, d=2, ms=5, mcs=10, eps=0.0, method=0, single=0, nl=0, seed=1, lab=P, prob=P,
        src=P, dst=P, w=P, nc=P, ws=P * 256, wsb=1 << 40):
    return L().b2d_hdbscan_rbc_fit(None, metric, x, ldx, m, d, ms, mcs, eps, method, single, nl, seed, lab, prob, src,
                                   dst, w, nc, ws, wsb)


NULLS = "null labels / probabilities / mst_src / mst_dst / mst_w / n_clusters"


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(metric=0), U, "hdbscan rbc supports the L2Unexpanded and L2SqrtUnexpanded metrics, got metric 0"),
    (dict(metric=1), U, "hdbscan rbc supports the L2Unexpanded and L2SqrtUnexpanded metrics, got metric 1"),
    (dict(m=0), E, "m must be positive and n_landmarks non-negative"),
    (dict(nl=-1), E, "m must be positive and n_landmarks non-negative"),
    (dict(d=4, ldx=4), U, "hdbscan rbc supports d = 2 and d = 3, got d = 4"),
    (dict(d=1, ldx=1), U, "hdbscan rbc supports d = 2 and d = 3, got d = 1"),
    (dict(m=2 ** 30), U, "hdbscan rbc: m must be below 2^30"),
    (dict(nl=101), E, "n_landmarks must be in [0, m] (0: ceil(sqrt(m)))"),
    (dict(x=None), E, "null x"),
    (dict(ldx=1), E, "leading dimension smaller than d"),
    (dict(ms=0), E, "min_samples must be in [1, min(64, m)], got 0"),
    (dict(ms=65), E, "min_samples must be in [1, min(64, m)], got 65"),
    (dict(m=3, ms=4), E, "min_samples must be in [1, min(64, m)], got 4"),
    (dict(mcs=1), E, "min_cluster_size must be at least 2, got 1"),
    (dict(eps=-0.5), E, "cluster_selection_epsilon must be finite and non-negative"),
    (dict(eps=float("nan")), E, "cluster_selection_epsilon must be finite and non-negative"),
    (dict(eps=float("inf")), E, "cluster_selection_epsilon must be finite and non-negative"),
    (dict(method=2), E, "method must be B2D_HDBSCAN_EOM or B2D_HDBSCAN_LEAF, got 2"),
    (dict(single=2), E, "allow_single_cluster must be 0 or 1"),
    (dict(lab=None), E, NULLS),
    (dict(prob=None), E, NULLS),
    (dict(src=None), E, NULLS),
    (dict(dst=None), E, NULLS),
    (dict(w=None), E, NULLS),
    (dict(nc=None), E, NULLS),
    (dict(ws=None, wsb=0), W, "workspace too small: need "),
    (dict(wsb=10), W, "workspace too small: need "),
    (dict(ws=P * 256 + 8), E, "workspace must be 256-byte aligned"),
])
def test_invalid_arguments(kw, rc, msg):
    assert fit(**kw) == rc, kw
    assert L().b2d_last_error().decode().startswith(msg)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert fit() == _lib.B2D_ERR_CUDA
    assert fit(m=1, ms=1, src=None, dst=None, w=None) == _lib.B2D_ERR_CUDA   # one row: no tree, the index still
    assert fit(d=3, ldx=5, metric=L2, method=1, single=1, eps=0.5) == _lib.B2D_ERR_CUDA


class FakeCuda:
    """an object with a __cuda_array_interface__ that is never read (the calls below fail in validation)"""

    def __init__(self, shape, strides=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (P, False), "version": 3,
                                         "strides": strides}


@pytest.mark.parametrize("kw,exc,msg", [
    (dict(metric="cosine"), _lib.LogicError, "hdbscan supports the euclidean and sqeuclidean metrics"),
    (dict(shape=(10, 4)), _lib.LogicError, "hdbscan supports d = 2 and d = 3, got d = 4"),
    (dict(n_landmarks=11), _lib.LogicError, "n_landmarks must be in [0, m]"),
    (dict(strides=(8, 8)), ValueError, "X must have contiguous rows"),
    (dict(min_cluster_size=1), _lib.LogicError, "min_cluster_size must be at least 2"),
    (dict(min_cluster_size=11), _lib.LogicError, "min_samples must be in [1, min(64, m)], got 11"),
    (dict(min_samples=0), _lib.LogicError, "min_samples must be in [1, min(64, m)], got 0"),
    (dict(shape=(100, 2), min_samples=65), _lib.LogicError, "min_samples must be in [1, min(64, m)], got 65"),
    (dict(cluster_selection_epsilon=-1.0), _lib.LogicError, "cluster_selection_epsilon must be finite and non-negative"),
    (dict(cluster_selection_epsilon=float("inf")), _lib.LogicError, "cluster_selection_epsilon must be finite"),
    (dict(cluster_selection_method="flat"), _lib.LogicError, "cluster_selection_method must be 'eom' or 'leaf'"),
])
def test_python_argument_errors(kw, exc, msg):
    from raft_b200.cluster import hdbscan
    kw = dict(kw)
    x = FakeCuda(kw.pop("shape", (10, 2)), strides=kw.pop("strides", None))
    with pytest.raises(exc, match=re.escape(msg)):
        hdbscan(x, handle=object(), **kw)


def test_python_signature():
    import inspect
    from raft_b200.cluster import HdbscanOutput, hdbscan
    params = list(inspect.signature(hdbscan).parameters.items())
    assert [(k, p.default) for k, p in params[1:]] == [
        ("min_cluster_size", 5), ("min_samples", None), ("cluster_selection_epsilon", 0.0),
        ("cluster_selection_method", "eom"), ("allow_single_cluster", False), ("metric", "euclidean"),
        ("n_landmarks", None), ("seed", 0), ("handle", None)]
    assert HdbscanOutput._fields == ("labels", "probabilities", "n_clusters", "mst")
