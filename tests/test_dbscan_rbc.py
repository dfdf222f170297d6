"""DBSCAN on the random ball cover without a GPU: the oracle of the GPU tier (tests/ball_cover_ref.dist(x, x) <= e fed to
tests/dbscan_ref.py) against sklearn.cluster.DBSCAN(metric="precomputed") and its bitwise symmetry on adversarial
points, the ABI declarations, every argument check of b2d_dbscan_rbc_fit with its status and message, B2D_ERR_CUDA
without a device, the recorded workspace contract (tests/golden/dbscan_rbc_workspace_contract.json), the Python
argument errors and the C++ shim's compile (its run on the GPU is in tests/test_dbscan_rbc_gpu.py)."""
import os
import re

import numpy as np
import pytest
import torch

import ball_cover_ref as bref
import cpp_build
from dbscan_ref import dbscan_ref
from raft_b200 import _lib
from test_workspace_contract import SIZE_MAX, load, replay_bytes, replay_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE
L2, L2SQRT = 4, 5   # L2Unexpanded, L2SqrtUnexpanded
NEW = ["b2d_dbscan_rbc_workspace_bytes", "b2d_dbscan_rbc_fit"]


def L():
    return _lib.lib()


def adjacency(x, eps, metric):
    """A of the contract for float32 points x (a torch tensor on any device): dist(x, x) <= fp32(eps)"""
    e = np.float32(eps)
    return (bref.dist(x, x, metric) <= float(e)).cpu().numpy()


def adversarial(kind, d, seed=5):
    """the ball cover tests' hard cases, sized for the CPU"""
    r = np.random.default_rng(seed)
    if kind == "lattice":   # eps at a lattice distance puts mass ties on the threshold
        g = np.stack(np.meshgrid(*[np.arange(7 if d == 3 else 18)] * d, indexing="ij"), -1).reshape(-1, d)
        return g.astype(np.float32)
    if kind == "duplicates":
        return r.random((37, d)).astype(np.float32)[r.integers(0, 37, 300)]
    if kind == "cancellation":   # a 1e4 offset with a 1e-2 spread
        return (1e4 + 1e-2 * r.random((300, d))).astype(np.float32)
    if kind == "subnormal":      # 1e-20 coordinates: subnormal squares
        return (1e-20 * r.random((300, d))).astype(np.float32)
    if kind == "dense_ball":     # one dense ball with sparse outliers
        return np.concatenate([1e-3 * r.random((280, d)), 1e3 * r.random((20, d))]).astype(np.float32)
    raise ValueError(kind)


KINDS = ["lattice", "duplicates", "cancellation", "subnormal", "dense_ball"]


def typical_eps(x, metric, q):
    dd = bref.dist(torch.from_numpy(x), torch.from_numpy(x), metric)
    pos = dd[dd > 0]
    return float(torch.quantile(pos.double(), q)) if pos.numel() else 1.0


@pytest.mark.parametrize("metric", ["sqeuclidean", "euclidean"])
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("kind", KINDS)
def test_adjacency_is_bitwise_symmetric(kind, d, metric):
    x = torch.from_numpy(adversarial(kind, d))
    dd = bref.dist(x, x, metric)
    assert torch.equal(dd.view(torch.int32), dd.t().contiguous().view(torch.int32))
    assert (torch.diagonal(dd) == 0).all()


@pytest.mark.parametrize("metric", ["sqeuclidean", "euclidean"])
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("kind", KINDS)
def test_oracle_equals_sklearn_precomputed(kind, d, metric):
    cluster = pytest.importorskip("sklearn.cluster")
    xn = adversarial(kind, d)
    x = torch.from_numpy(xn)
    dd = bref.dist(x, x, metric).double().numpy()
    if kind == "lattice":
        eps_list = [1.0, 2.0] if metric == "sqeuclidean" else [1.0, float(np.float32(np.sqrt(np.float32(2))))]
    else:
        eps_list = [typical_eps(xn, metric, 0.01), typical_eps(xn, metric, 0.1)]
    for eps in eps_list:
        A = adjacency(x, eps, metric)
        for ms in (1, 2, 5, 20, len(xn) + 1):
            sk = cluster.DBSCAN(eps=float(np.float32(eps)), min_samples=ms, metric="precomputed").fit(dd)
            lab, csi, nc = dbscan_ref(A, ms)
            assert (lab == sk.labels_).all(), (kind, eps, ms)
            ncore = len(sk.core_sample_indices_)
            assert (csi[:ncore] == sk.core_sample_indices_).all() and (csi[ncore:] == -1).all()
            assert nc == len(set(sk.labels_.tolist()) - {-1})


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(L(), s)
    assert "b2d_dbscan_fit(" in hdr   # the brute fit stays as it is


def test_workspace_queries():
    for args in ((-1, 2, 0), (2 ** 31, 2, 0), (10, 1, 0), (10, 4, 0), (10, 2, -1), (10, 2, 11)):
        assert L().b2d_dbscan_rbc_workspace_bytes(*args) == SIZE_MAX, args
    for m, d in ((1, 2), (1000, 3), (10 ** 6, 2)):
        full = L().b2d_dbscan_rbc_workspace_bytes(m, d, 0)
        index = L().b2d_ball_cover_index_bytes(m, d, 0)
        build = L().b2d_ball_cover_build_workspace_bytes(m, d, 0)
        # the index, then the build's scratch, which the fit's five [m] arrays overlap
        assert full >= index + max(build, 20 * m)
        assert full <= index + max(build, 20 * m + 8192)
        assert L().b2d_dbscan_rbc_workspace_bytes(m, d, int(np.ceil(np.sqrt(m)))) == full
    assert L().b2d_dbscan_rbc_workspace_bytes(0, 2, 0) != SIZE_MAX


def test_workspace_contract_bytes():
    c = load("dbscan_rbc_workspace_contract.json")
    for m, d, nl, want in replay_bytes(c, "b2d_dbscan_rbc_workspace_bytes"):
        assert (want == SIZE_MAX) == (not (0 <= m < 2 ** 31 and d in (2, 3) and 0 <= nl <= m)), (m, d, nl)


def test_workspace_contract_errors():
    assert replay_errors(load("dbscan_rbc_workspace_contract.json")) == 2 * 2 * 3


def fit(metric=L2SQRT, x=P, ldx=2, m=100, d=2, eps=0.5, ms=5, nl=0, seed=1, lab=P, csi=P, ncl=P, ws=P * 256,
        wsb=1 << 40):
    return L().b2d_dbscan_rbc_fit(None, metric, x, ldx, m, d, eps, ms, nl, seed, lab, csi, ncl, ws, wsb)


MSG_METRIC = "dbscan rbc supports the L2Unexpanded and L2SqrtUnexpanded metrics, got metric %d"


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(metric=0), U, MSG_METRIC % 0),
    (dict(metric=1), U, MSG_METRIC % 1),
    (dict(metric=2), U, MSG_METRIC % 2),
    (dict(metric=-1), U, MSG_METRIC % -1),
    (dict(metric=13), U, MSG_METRIC % 13),
    (dict(m=-1), E, "negative extent or n_landmarks"),
    (dict(nl=-1), E, "negative extent or n_landmarks"),
    (dict(m=2 ** 31), E, "dbscan: m must be below 2^31"),
    (dict(d=1, ldx=1), U, "dbscan rbc supports d = 2 and d = 3, got d = 1"),
    (dict(d=4, ldx=4), U, "dbscan rbc supports d = 2 and d = 3, got d = 4"),
    (dict(d=0), U, "dbscan rbc supports d = 2 and d = 3, got d = 0"),
    (dict(nl=101), E, "n_landmarks must be in [0, m] (0: ceil(sqrt(m)))"),
    (dict(ms=0), E, "min_samples must be >= 1"),
    (dict(ms=-3), E, "min_samples must be >= 1"),
    (dict(x=None), E, "null x / labels"),
    (dict(lab=None), E, "null x / labels"),
    (dict(ldx=1), E, "leading dimension smaller than d"),
    (dict(d=3, ldx=2), E, "leading dimension smaller than d"),
    (dict(ws=None, wsb=0), W, "workspace too small: need "),
    (dict(wsb=10), W, "workspace too small: need "),
    (dict(ws=P * 256 + 8), E, "workspace must be 256-byte aligned"),
])
def test_fit_invalid_arguments(kw, rc, msg):
    assert fit(**kw) == rc, kw
    assert L().b2d_last_error().decode().startswith(msg)


def test_fit_empty_is_a_noop():
    # m == 0 touches nothing, whatever the pointers
    assert fit(m=0, x=None, lab=None, csi=None, ncl=None, ws=None, wsb=0) == _lib.B2D_OK
    assert fit(m=0, d=3, ldx=3, eps=float("nan")) == _lib.B2D_OK


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert fit() == _lib.B2D_ERR_CUDA
    assert fit(d=3, ldx=5, metric=L2, csi=None, ncl=None) == _lib.B2D_ERR_CUDA
    for eps in (float("nan"), -1.0, float("inf"), 0.0):   # every eps still enqueues work: the index and the labels
        assert fit(eps=eps) == _lib.B2D_ERR_CUDA


class FakeCuda:
    """an object with a __cuda_array_interface__ that is never read (the calls below fail in validation)"""

    def __init__(self, shape, typestr="<f4", strides=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (P, False), "version": 3,
                                         "strides": strides}


@pytest.mark.parametrize("kw,exc,msg", [
    (dict(metric="cosine"), _lib.LogicError, "supports the euclidean and sqeuclidean metrics"),
    (dict(shape=(10, 4)), _lib.LogicError, "supports d = 2 and d = 3, got d = 4"),
    (dict(shape=(10, 1)), _lib.LogicError, "supports d = 2 and d = 3, got d = 1"),
    (dict(max_mbytes_per_batch=64), _lib.LogicError, "has no batches"),
    (dict(n_landmarks=11), _lib.LogicError, "n_landmarks must be in [0, m]"),
    (dict(n_landmarks=-1), _lib.LogicError, "n_landmarks must be in [0, m]"),
    (dict(min_samples=0), _lib.LogicError, "min_samples must be >= 1"),
    (dict(algorithm="kd_tree"), _lib.LogicError, "algorithm must be 'brute' or 'rbc'"),
    (dict(metric="manhattan"), _lib.LogicError, "dbscan supports the euclidean, sqeuclidean and cosine metrics"),
])
def test_python_argument_errors(kw, exc, msg):
    from raft_b200.cluster import dbscan
    kw = dict(kw)
    x = FakeCuda(kw.pop("shape", (10, 2)))
    args = dict(algorithm="rbc")
    args.update(kw)
    with pytest.raises(exc, match=re.escape(msg)):
        dbscan(x, 0.5, handle=object(), **args)


def test_python_signature():
    import inspect
    from raft_b200.cluster import dbscan
    params = list(inspect.signature(dbscan).parameters.items())
    assert [(k, p.default) for k, p in params[2:]] == [
        ("min_samples", 5), ("metric", "euclidean"), ("max_mbytes_per_batch", None), ("algorithm", "brute"),
        ("n_landmarks", None), ("seed", 0), ("handle", None)]


def test_shim_compiles(tmp_path):
    for mock in (False, True):
        exe = str(tmp_path / ("dbscan_rbc_shim_mockraft" if mock else "dbscan_rbc_shim"))
        assert os.path.exists(cpp_build.build("dbscan_rbc_shim_test.cu", exe, mock))
